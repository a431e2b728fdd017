"""Thin Python wrappers over the C ABI's kernel-level entry points (PyTorch tensors in/out).

Random ops consume the torch CUDA generator exactly like the torch ops they replace: they read
(seed, philox offset) from the generator, run the kernel on that stream, and advance the offset by
what the torch kernel would have consumed (ATen/native/cuda/DistributionTemplates.h:50-62).
"""
from __future__ import annotations

import math
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


# ------------------------------------------------------------------ top-k / top-p truncation
# The fused sampler keeps, per token, the top-k codes and then the smallest top set holding a fraction top-p of the probability
# (include/paella_b200.h, pb200_paella_sample_tokens_params_trunc); the draw is otherwise unchanged.  The kernels read a device
# table of int32 k [B] and float32 p [B], 0 and 1.0 meaning off.
def _truncation_values(name: str, value, batch: int, is_k: bool) -> list:
    if value is None:
        return [None] * batch
    if torch.is_tensor(value):
        if value.device.type != "cpu":
            raise ValueError(f"{name}: per-sample values must be a CPU tensor (got {value.device}; reading it would synchronise the stream)")
        if tuple(value.shape) != (batch,):
            raise ValueError(f"{name}: per-sample values of shape {list(value.shape)} for a batch of {batch} (expected [{batch}])")
        if is_k and (value.is_floating_point() or value.is_complex() or value.dtype == torch.bool):
            raise ValueError(f"{name}: per-sample values must be an integer tensor (got {value.dtype})")
        if not is_k and not value.is_floating_point():
            raise ValueError(f"{name}: per-sample values must be a floating-point tensor (got {value.dtype})")
        vals = value.tolist()
    else:
        if is_k and (isinstance(value, bool) or not isinstance(value, int)):
            raise ValueError(f"{name}={value!r}: expected None, an int >= 0 or a CPU integer tensor [{batch}]")
        if not is_k and (isinstance(value, bool) or not isinstance(value, (int, float))):
            raise ValueError(f"{name}={value!r}: expected None, a float in (0, 1] or a CPU float tensor [{batch}]")
        vals = [value] * batch
    for v in vals:
        if is_k and v < 0:
            raise ValueError(f"{name}: every k must be >= 0 (0 is off; got {vals})")
        if not is_k and not 0.0 < v <= 1.0:        # NaN fails this too
            raise ValueError(f"{name}: every p must be in (0, 1] (1.0 is off; got {vals})")
    return vals


def truncation_table(top_k, top_p, batch: int, num_labels: int) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
    """``top_k`` (None, an int >= 0, or a CPU integer tensor [batch]) and ``top_p`` (None, a float in (0, 1], or a CPU float
    tensor [batch]) as the host truncation table: (int32 k [batch], float32 p [batch]), with k = 0 where the row keeps every
    code (None, 0 or k >= num_labels) and p = 1.0 where it does (None or 1.0).  None when no row truncates.  ValueError, before
    anything is enqueued, for a non-integer or negative k, a p <= 0, > 1 or NaN, a CUDA tensor, or a wrong shape."""
    ks = _truncation_values("top_k", top_k, batch, True)
    ps = _truncation_values("top_p", top_p, batch, False)
    k = torch.tensor([0 if v is None or v >= num_labels else int(v) for v in ks], dtype=torch.int32)
    p = torch.tensor([1.0 if v is None else float(v) for v in ps], dtype=torch.float32)
    if not bool((k > 0).any()) and not bool((p < 1.0).any()):
        return None
    return k, p


# ------------------------------------------------------------------ seamless tiling
# The denoiser's ResBlock depthwise convolutions and the decoder's ReplicationPad2d / ConvTranspose2d read across a wrapped edge
# (include/paella_b200.h, pb200_paella_features_tiled, pb200_vqgan_decode_tiled).  The kernels read a device table of one byte per
# sample: bit 0 wraps x (left and right edges), bit 1 wraps y (top and bottom).
TILINGS = {None: 0, "none": 0, "x": 1, "y": 2, "xy": 3}


def _tiling_code(name: str, value) -> int:
    if not (value is None or isinstance(value, str)) or value not in TILINGS:
        raise ValueError(f"{name}={value!r}: expected None, 'none', 'x', 'y' or 'xy'")
    return TILINGS[value]


def tiling_codes(tiling, batch: int) -> list:
    """``tiling`` (one value for every sample, or a list or tuple of ``batch`` values) -> the ``batch`` wrap codes.  ValueError,
    before anything is enqueued, for an unknown value, a list of the wrong length, or a tensor."""
    if isinstance(tiling, (list, tuple)):
        if len(tiling) != batch:
            raise ValueError(f"tiling: got {len(tiling)} entries for a batch of {batch} (one per sample)")
        return [_tiling_code(f"tiling[{b}]", v) for b, v in enumerate(tiling)]
    if torch.is_tensor(tiling):
        raise ValueError("tiling: expected None, 'none', 'x', 'y', 'xy' or a list of them (got a tensor)")
    return [_tiling_code("tiling", tiling)] * batch


def tiling_table(tiling, batch: int) -> Optional[torch.Tensor]:
    """``tiling`` as the host wrap table: uint8 [batch], or None when no sample wraps (the call then launches exactly the
    zero- / replication-padding kernels).  ValueError as in ``tiling_codes``."""
    codes = tiling_codes(tiling, batch)
    return torch.tensor(codes, dtype=torch.uint8) if any(codes) else None


# ------------------------------------------------------------------ regional prompts
# Each sample may carry up to MAX_PROMPT_REGIONS (inputs, region) pairs.  Token t of a sample gets a mask byte: bit k >= 1 set iff
# t lies in region k, bit 0 iff it lies in no region.  The denoiser's AttnBlock positions OR their footprint's bytes and attend to
# the conditioning of every prompt they have a bit of, prompt 0 being the sample's own (include/paella_b200.h,
# pb200_paella_features_regional).
MAX_PROMPT_REGIONS = 7


def check_conditioning_inputs(name: str, inputs) -> None:
    """ValueError unless ``inputs`` is a batch-1 conditioning dict: ``byt5`` [1, L, byt5_embd] with L >= 1, and optional ``clip``
    and ``clip_image`` (a tensor or a list or tuple of tensors) whose first dimension is 1."""
    if not isinstance(inputs, dict) or not torch.is_tensor(inputs.get("byt5")):
        raise ValueError(f"{name}: expected a conditioning dict with a 'byt5' tensor (got {type(inputs).__name__})")
    byt5 = inputs["byt5"]
    if byt5.dim() != 3 or byt5.shape[0] != 1 or byt5.shape[1] < 1:
        raise ValueError(f"{name}: byt5 of shape {list(byt5.shape)}; expected [1, L, byt5_embd] with L >= 1")
    ci = inputs.get("clip_image")
    extra = [("clip", inputs.get("clip"))] + [("clip_image", t) for t in (ci if isinstance(ci, (list, tuple)) else [ci])]
    for key, t in extra:
        if t is not None and (not torch.is_tensor(t) or t.dim() < 1 or t.shape[0] != 1):
            raise ValueError(f"{name}: {key} must be None or a tensor of batch 1")


def regional_table(prompt_regions, batch: int, hw, device=None):
    """``prompt_regions`` (None, or a list or tuple of ``batch`` entries, each None or a list or tuple of at most
    MAX_PROMPT_REGIONS (inputs, region) pairs) -> None when no sample has a region, otherwise (uint8 [batch, H, W] token masks,
    the list of each sample's region inputs in order).  ``inputs``: a batch-1 conditioning dict; ``region``: a bool [H, W]
    tensor on the CPU or on ``device`` (copied to the host).  A single pair or list of pairs is not broadcast.  ValueError
    for any other shape of the argument, before anything is enqueued."""
    if prompt_regions is None:
        return None
    if not isinstance(prompt_regions, (list, tuple)):
        raise ValueError(f"prompt_regions: expected None or a list of {batch} entries (got {type(prompt_regions).__name__})")
    if len(prompt_regions) != batch:
        raise ValueError(f"prompt_regions: got {len(prompt_regions)} entries for a batch of {batch} (one per sample, None for none)")
    H, W = int(hw[0]), int(hw[1])
    masks = torch.zeros(batch, H, W, dtype=torch.uint8)
    prompts = []
    for b, entry in enumerate(prompt_regions):
        if entry is None:
            entry = []
        if not isinstance(entry, (list, tuple)):
            raise ValueError(f"prompt_regions[{b}]: expected None or a list of (inputs, region) pairs (got {type(entry).__name__})")
        if len(entry) > MAX_PROMPT_REGIONS:
            raise ValueError(f"prompt_regions[{b}]: {len(entry)} regions; at most {MAX_PROMPT_REGIONS}")
        own = []
        for k, pair in enumerate(entry, start=1):
            name = f"prompt_regions[{b}][{k - 1}]"
            if not isinstance(pair, (list, tuple)) or len(pair) != 2:
                raise ValueError(f"{name}: expected an (inputs, region) pair")
            inputs, region = pair
            check_conditioning_inputs(name, inputs)
            if not torch.is_tensor(region) or region.dtype != torch.bool or tuple(region.shape) != (H, W):
                raise ValueError(f"{name}: region must be a bool tensor of shape [{H}, {W}]")
            if region.device.type != "cpu" and (device is None or region.device != torch.device(device)):
                raise ValueError(f"{name}: region is on {region.device}, the model on {device}")
            masks[b] |= region.cpu().to(torch.uint8) << k
            own.append(inputs)
        masks[b][masks[b] == 0] = 1
        prompts.append(own)
    if not any(prompts):
        return None
    return masks, prompts


def check_regions_unweighted(table, attn_weights) -> None:
    """ValueError if a sample of regional_table's ``table`` has regions and ``attn_weights`` (one vector for every sample, or a
    list with an entry per sample) weights it: the two are not defined together."""
    if table is None or attn_weights is None:
        return
    for b, own in enumerate(table[1]):
        if own and (not isinstance(attn_weights, (list, tuple)) or attn_weights[b] is not None):
            raise ValueError(f"prompt_regions[{b}]: regional prompts and attn_weights on one sample are not supported")


def check_attention_maps(attention_maps, prompt_regions=None) -> bool:
    """``attention_maps`` -> the flag.  ValueError, before anything is enqueued, unless it is a bool, and for maps on a call or
    request that also has ``prompt_regions``: regional tiles gate the sample's own prompt keys per query, and maps are not
    defined there."""
    if not isinstance(attention_maps, bool):
        raise ValueError(f"attention_maps: expected a bool (got {type(attention_maps).__name__})")
    if attention_maps and prompt_regions is not None:
        raise ValueError("attention_maps: not defined together with prompt_regions")
    return attention_maps


# ------------------------------------------------------------------ prompt-to-prompt editing
# Sample b with attention_source[b] = (a, k) replays sample a's attention probabilities in its conditional forward on steps i < k,
# in every AttnBlock and head, with its own values and attn_weights (pb200_paella_features_inject).  The table holds, per step, the
# source of each sample or -1.
def _is_int(v) -> bool:
    return isinstance(v, int) and not isinstance(v, bool)


def attention_source_table(attention_source, batch: int, steps: int, regions=None, exact: bool = False,
                           forward: bool = False) -> Optional[torch.Tensor]:
    """``attention_source`` (None, or a list or tuple of ``batch`` entries, each None or an (a, k) pair of ints; with ``forward``
    each None or an int a, injected in that single forward) -> None when no sample is injected on any step, otherwise int32 CPU
    [steps, batch]: entry [i, b] is a when i < k, else -1.  ``regions``: regional_table's result, whose samples with regions may be
    neither sources nor edits.  ValueError, before anything is enqueued, for the wrong length, a bad entry (a bool is not an int),
    a source out of range or equal to its sample, a source that is itself injected, k outside [0, steps], regions on an edit or
    its source, and ``exact=True``."""
    if attention_source is None:
        return None
    if not isinstance(attention_source, (list, tuple)):
        raise ValueError(f"attention_source: expected None or a list of {batch} entries (got {type(attention_source).__name__})")
    if len(attention_source) != batch:
        raise ValueError(f"attention_source: got {len(attention_source)} entries for a batch of {batch} (one per sample, None for none)")
    pairs = []
    for b, entry in enumerate(attention_source):
        if entry is None:
            pairs.append(None)
            continue
        if forward:
            if not _is_int(entry):
                raise ValueError(f"attention_source[{b}]: expected None or the int index of a source sample (got {entry!r})")
            a, k = entry, steps
        else:
            if not isinstance(entry, (list, tuple)) or len(entry) != 2 or not _is_int(entry[0]) or not _is_int(entry[1]):
                raise ValueError(f"attention_source[{b}]: expected None or an (int source, int steps) pair (got {entry!r})")
            a, k = entry
        if not 0 <= a < batch or a == b:
            raise ValueError(f"attention_source[{b}]: source {a} is not another sample of the call (0..{batch - 1})")
        if not 0 <= k <= steps:
            raise ValueError(f"attention_source[{b}]: {k} injected steps; expected 0..{steps}")
        pairs.append((a, k))
    for b, p in enumerate(pairs):
        if p is not None and pairs[p[0]] is not None:
            raise ValueError(f"attention_source[{b}]: source {p[0]} is itself injected (no chains)")
        if p is not None and regions is not None and (regions[1][b] or regions[1][p[0]]):
            raise ValueError(f"attention_source[{b}]: prompt_regions on an injected sample or on its source are not supported")
    if all(p is None for p in pairs):
        return None
    if exact:
        raise ValueError("exact=True restates the reference op for op, which has no attention injection")
    table = torch.full((steps, batch), -1, dtype=torch.int32)
    for b, p in enumerate(pairs):
        if p is not None:
            table[:p[1], b] = p[0]
    return table


# ------------------------------------------------------------------ LoRA adapters
# Each sample may run under one LoRA adapter at a scale (paella_b200/lora.py): its rows get the adapter's deltas in every AttnBlock
# (pb200_paella_features_lora) and its conditioning slots are projected under it (pb200_paella_prepare_cond_lora).
MAX_LORA_ADAPTERS = 32


def _lora_entry(name: str, entry, model):
    """None, an adapter or (adapter, scale) -> None or (adapter, scale); a scale of 0 is None.  ValueError for anything else, a
    non-finite scale, and an adapter packed for another configuration or on another device."""
    from .lora import LoraAdapter
    if entry is None:
        return None
    if isinstance(entry, LoraAdapter):
        adapter, scale = entry, 1.0
    elif isinstance(entry, (list, tuple)) and len(entry) == 2 and isinstance(entry[0], LoraAdapter):
        adapter, scale = entry
        if isinstance(scale, bool) or not isinstance(scale, (int, float)):
            raise ValueError(f"{name}: the scale must be a real number (got {scale!r})")
        scale = float(scale)
        if not math.isfinite(scale):
            raise ValueError(f"{name}: the scale must be finite (got {scale!r})")
    else:
        raise ValueError(f"{name}: expected None, a LoraAdapter or an (adapter, scale) pair (got {type(entry).__name__})")
    if adapter.config != model._cfg:
        raise ValueError(f"{name}: the adapter was loaded for another model configuration")
    if adapter.device != model._device():
        raise ValueError(f"{name}: the adapter is on {adapter.device}, the model on {model._device()}")
    return None if scale == 0.0 else (adapter, scale)


def _is_lora_entry(lora) -> bool:
    from .lora import LoraAdapter
    return isinstance(lora, LoraAdapter) or (isinstance(lora, tuple) and len(lora) == 2 and isinstance(lora[0], LoraAdapter))


def lora_table(lora, batch: int, model):
    """``lora`` (None; an adapter or (adapter, scale) for every sample; or a list or tuple of ``batch`` such entries, each also
    possibly None) -> None when no sample runs under an adapter, otherwise (adapters, ids, scales): the distinct adapters in order
    of first use, int32 CPU [batch] of each sample's index into them (-1: none) and float32 CPU [batch] scales (0 where none).
    ValueError, before anything is enqueued, for the wrong length, a bad entry or scale, an adapter of another configuration or
    device, and more than 32 distinct adapters."""
    if lora is None:
        return None
    if _is_lora_entry(lora):
        entries = [_lora_entry("lora", lora, model)] * batch
    elif isinstance(lora, (list, tuple)):
        if len(lora) != batch:
            raise ValueError(f"lora: got {len(lora)} entries for a batch of {batch} (one per sample, None for none)")
        entries = [_lora_entry(f"lora[{b}]", e, model) for b, e in enumerate(lora)]
    else:
        raise ValueError(f"lora: expected None, a LoraAdapter, an (adapter, scale) pair or a list of {batch} entries "
                         f"(got {type(lora).__name__})")
    table = lora_rows(entries)
    return table if table[0] else None


def distinct_adapters(entries) -> list:
    """The distinct adapters of per-row entries (None or (adapter, scale)), in order of first use."""
    adapters = []
    for e in entries:
        if e is not None and not any(a is e[0] for a in adapters):
            adapters.append(e[0])
    return adapters


def lora_rows(entries):
    """Per-row entries (None or (adapter, scale)) -> (adapters, ids, scales): the distinct adapters in order of first use, int32 CPU
    [rows] of each row's index into them (-1: none) and float32 CPU [rows] scales (0 where none) -- the index space of one launch's
    adapter array.  ValueError for more than MAX_LORA_ADAPTERS distinct adapters."""
    adapters = distinct_adapters(entries)
    if len(adapters) > MAX_LORA_ADAPTERS:
        raise ValueError(f"lora: {len(adapters)} distinct adapters in one call (at most {MAX_LORA_ADAPTERS})")
    ids = torch.tensor([-1 if e is None else next(i for i, a in enumerate(adapters) if a is e[0]) for e in entries], dtype=torch.int32)
    scales = torch.tensor([0.0 if e is None else e[1] for e in entries], dtype=torch.float32)
    return adapters, ids, scales


def lora_entries(table, batch: int) -> list:
    """lora_table's result -> per sample None or (adapter, scale)."""
    if table is None:
        return [None] * batch
    adapters, ids, scales = table
    return [None if i < 0 else (adapters[i], float(s)) for i, s in zip(ids.tolist(), scales.tolist())]


def lora_rows_to_device(entries, device):
    """lora_rows on per-row entries, the two tables in one asynchronous copy: (adapters, device int32 ids, device float32 scales)."""
    adapters, ids, scales = lora_rows(entries)
    ids_d, scales_d = to_device_packed([ids, scales], device)
    return adapters, ids_d, scales_d


def lora_device(table, device):
    """lora_table's result -> Paella.features' ``lora``: (HOST adapter array, its length, device int32 ids, device float32 scales),
    the two tables in one asynchronous copy; None stays None."""
    if table is None:
        return None
    adapters, ids, scales = table
    ids_d, scales_d = to_device_packed([ids, scales], device)
    return lora_structs(adapters), len(adapters), ids_d, scales_d


def lora_structs(adapters):
    """The HOST pb200_lora_adapter array of a table's adapters."""
    arr = (_lib.LoraAdapter * max(1, len(adapters)))()
    for i, a in enumerate(adapters):
        arr[i] = a._c
    return arr


# ------------------------------------------------------------------ guidance prompts
# Each sample of a guided call may carry up to MAX_GUIDANCE_PROMPTS (inputs, weight) terms.  On a guided step with scale cfg its
# logits are l_u + cfg * [(l_c - l_u) + sum_j w_j (l_j - l_u)], l_j being the conditional forward under term j's inputs.  The
# coefficients (a_c, a_u, a_1 ..) sum to 1, so the mix runs on the features before the out_mapper GEMM
# (pb200_paella_guidance_mix), and the sampler then takes the mixed row with (1, 0, 1/T).
MAX_GUIDANCE_PROMPTS = 7


def guidance_table(guidance_prompts, batch: int):
    """``guidance_prompts`` (None, or a list or tuple of ``batch`` entries, each None or a list or tuple of at most
    MAX_GUIDANCE_PROMPTS (inputs, weight) pairs) -> None when no sample has a term, otherwise the ``batch`` lists of (inputs,
    float weight) pairs.  ``inputs``: a batch-1 conditioning dict (check_conditioning_inputs); ``weight``: a finite real number,
    negative for a further negative prompt.  ValueError for any other shape of the argument, before anything is enqueued."""
    if guidance_prompts is None:
        return None
    if not isinstance(guidance_prompts, (list, tuple)):
        raise ValueError(f"guidance_prompts: expected None or a list of {batch} entries (got {type(guidance_prompts).__name__})")
    if len(guidance_prompts) != batch:
        raise ValueError(f"guidance_prompts: got {len(guidance_prompts)} entries for a batch of {batch} (one per sample, None for none)")
    terms = []
    for b, entry in enumerate(guidance_prompts):
        if entry is None:
            entry = []
        if not isinstance(entry, (list, tuple)):
            raise ValueError(f"guidance_prompts[{b}]: expected None or a list of (inputs, weight) pairs (got {type(entry).__name__})")
        if len(entry) > MAX_GUIDANCE_PROMPTS:
            raise ValueError(f"guidance_prompts[{b}]: {len(entry)} terms; at most {MAX_GUIDANCE_PROMPTS}")
        own = []
        for j, pair in enumerate(entry):
            name = f"guidance_prompts[{b}][{j}]"
            if not isinstance(pair, (list, tuple)) or len(pair) != 2:
                raise ValueError(f"{name}: expected an (inputs, weight) pair")
            inputs, weight = pair
            check_conditioning_inputs(name, inputs)
            if isinstance(weight, bool) or not isinstance(weight, (int, float)) or not math.isfinite(weight):
                raise ValueError(f"{name}: weight must be a finite real number (got {weight!r})")
            own.append((inputs, float(weight)))
        terms.append(own)
    if not any(terms):
        return None
    return terms


def guidance_coefficients(cfg: float, weights, pag: float = 0.0) -> list:
    """The mix coefficients of one guided step as fp32 values: (float)(cfg + s), (float)(1 - cfg (1 + sum w)), then (float)(cfg w_j)
    per term, then (float)(-s) for a perturbed row (pag = s != 0), from doubles.  With no terms and no PAG they are (cfg, 1 - cfg)
    of sampling_params, bit for bit.  ``cfg`` None (an unguided sample): (1 + s, -s), the mix l_c + s (l_c - l_p)."""
    s = float(pag)
    if cfg is None:
        vals = [1.0 + s, -s]
    else:
        c = float(cfg)
        total = 0.0
        for w in weights:
            total += w
        vals = [c + s, 1.0 - c * (1.0 + total)] + [c * w for w in weights] + ([-s] if s != 0.0 else [])
    return torch.tensor(vals, dtype=torch.float64).float().tolist()


def guidance_mix_table(terms, cond_row, uncond_row, term_rows, cfgs, pag=None, pag_row=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """The per-call mix table of the composed samples (those with terms or PAG, in ``terms`` order of the samples given): int32
    [n_composed, 2 + J] row indices [c, u, t_1 .. t_J, p] (-1 after a sample's last row) and float32 [steps, n_composed, 2 + J]
    coefficients (guidance_coefficients, 0 after the last row).  ``terms``: each composed sample's weights; ``cond_row``,
    ``uncond_row``: its rows (uncond_row None: an unguided call, rows [c, p]); ``term_rows``: its term rows; ``cfgs``: per step, each
    composed sample's cfg (None entries in an unguided call); ``pag``: None or each composed sample's PAG scale (0: none), with
    ``pag_row`` its perturbed row."""
    n = len(terms)
    pag = pag if pag is not None else [0.0] * n
    ld = max((1 if uncond_row is None else 2) + len(w) + (s != 0.0) for w, s in zip(terms, pag))
    rows = torch.full((n, ld), -1, dtype=torch.int32)
    coef = torch.zeros(len(cfgs), n, ld, dtype=torch.float32)
    for y, (ws, s) in enumerate(zip(terms, pag)):
        own = [cond_row[y]] + ([uncond_row[y]] if uncond_row is not None else []) + list(term_rows[y]) + ([pag_row[y]] if s != 0.0 else [])
        rows[y, :len(own)] = torch.tensor(own, dtype=torch.int32)
        for i, step_cfgs in enumerate(cfgs):
            coef[i, y, :len(own)] = torch.tensor(guidance_coefficients(step_cfgs[y], ws, s))
    return rows, coef


# ------------------------------------------------------------------ perturbed-attention guidance
# A sample may carry a PAG entry (s, blocks): its perturbed forward is its conditional forward with the self part of every
# attention map of the AttnBlocks in ``blocks`` (plan order, paella_b200.lora.attn_blocks) collapsed onto the diagonal
# (pb200_attention_perturb), and its guided logits gain s (l_c - l_p) (Ahn et al. 2024, "Self-Rectifying Diffusion Sampling with
# Perturbed-Attention Guidance").  The perturbed forward is one more tail row that reads its sample's own conditioning slot; the
# per-row table of AttnBlock bit masks rides in the call's single packed copy (pb200_paella_features_pag).
MAX_PAG_BLOCKS = 64


def pag_default_blocks(cfg: dict) -> list:
    """The default perturbed AttnBlocks of a Paella configuration: those of the deepest level, down and up, in plan order."""
    from .lora import attn_blocks
    deepest = len(cfg["c_hidden"]) - 1
    return [i for i, (path, _) in enumerate(attn_blocks(cfg)) if path.startswith(f"down_blocks.{deepest}.") or path.startswith("up_blocks.0.")]


def _pag_blocks(name: str, blocks, n_blocks: int) -> int:
    """A non-empty list, tuple or set of distinct int AttnBlock indices in [0, n_blocks) -> its bit mask."""
    if not isinstance(blocks, (list, tuple, set, frozenset)) or len(blocks) == 0:
        raise ValueError(f"{name}: the blocks must be a non-empty list of AttnBlock indices (got {blocks!r})")
    mask = 0
    for i in blocks:
        if not _is_int(i):
            raise ValueError(f"{name}: AttnBlock index {i!r} is not an int")
        if not 0 <= i < n_blocks:
            raise ValueError(f"{name}: AttnBlock index {i} out of range (the model has {n_blocks} AttnBlocks)")
        if (mask >> i) & 1:
            raise ValueError(f"{name}: AttnBlock index {i} given twice")
        mask |= 1 << i
    return mask


def _pag_entry(name: str, entry, n_blocks: int, default_blocks):
    """None, a scale or (scale, blocks) -> (float scale, bit mask); a scale of 0 is no entry, (0.0, 0)."""
    if entry is None:
        return 0.0, 0
    if isinstance(entry, (list, tuple)):
        if len(entry) != 2:
            raise ValueError(f"{name}: expected None, a scale or a (scale, blocks) pair (got {entry!r})")
        scale, blocks = entry
    else:
        scale, blocks = entry, default_blocks
    if isinstance(scale, bool) or not isinstance(scale, (int, float)) or not math.isfinite(scale):
        raise ValueError(f"{name}: the scale must be a finite real number (got {scale!r})")
    mask = _pag_blocks(name, blocks, n_blocks)
    return (0.0, 0) if float(scale) == 0.0 else (float(scale), mask)


def _mask_i64(m: int) -> int:
    return m - (1 << 64) if m >= 1 << 63 else m


def pag_table(pag, batch: int, n_blocks: int, default_blocks=None, regions=None, inject=None, exact: bool = False,
              forward: bool = False):
    """``pag`` (None, or a list or tuple of ``batch`` entries, each None, a scale or a (scale, blocks) pair; with ``forward`` each
    None or a blocks list, perturbed in that single forward) -> None when no sample is perturbed, otherwise (scales, masks): the
    float scale of every sample (0: none; 1.0 with ``forward``) and the int64 CPU [batch] AttnBlock bit masks the kernels read as
    uint64 (0: none).  ``default_blocks``: the blocks of an entry given as a scale (pag_default_blocks).  ``regions``:
    regional_table's result; ``inject``: attention_source_table's result.  ValueError, before anything is enqueued, for the wrong
    length, a non-finite or bool scale, empty, duplicated, non-int or out-of-range blocks, more than 64 AttnBlocks, PAG on a sample
    with prompt_regions or on a prompt-to-prompt edit or source, and ``exact=True``."""
    if pag is None:
        return None
    if not isinstance(pag, (list, tuple)):
        raise ValueError(f"pag: expected None or a list of {batch} entries (got {type(pag).__name__})")
    if len(pag) != batch:
        raise ValueError(f"pag: got {len(pag)} entries for a batch of {batch} (one per sample, None for none)")
    if n_blocks > MAX_PAG_BLOCKS:
        raise ValueError(f"pag: the model has {n_blocks} AttnBlocks; the perturbation masks hold {MAX_PAG_BLOCKS}")
    if forward:
        entries = [(0.0, 0) if e is None else (1.0, _pag_blocks(f"pag_blocks[{b}]", e, n_blocks)) for b, e in enumerate(pag)]
    else:
        entries = [_pag_entry(f"pag[{b}]", e, n_blocks, default_blocks) for b, e in enumerate(pag)]
    edits = set()
    if inject is not None:
        for b in range(batch):
            col = inject[:, b]
            if bool((col >= 0).any()):
                edits.add(b)
                edits.update(int(a) for a in col[col >= 0].tolist())
    for b, (s, _) in enumerate(entries):
        if s == 0.0:
            continue
        if regions is not None and regions[1][b]:
            raise ValueError(f"pag[{b}]: perturbed-attention guidance on a sample with prompt_regions is not supported")
        if b in edits:
            raise ValueError(f"pag[{b}]: perturbed-attention guidance on a prompt-to-prompt edit or source is not supported")
    if all(s == 0.0 for s, _ in entries):
        return None
    if exact:
        raise ValueError("exact=True restates the reference op for op, which has no perturbed-attention guidance")
    return [s for s, _ in entries], torch.tensor([_mask_i64(m) for _, m in entries], dtype=torch.int64)


# ------------------------------------------------------------------ confidence-guided renoising
MAX_CONFIDENCE_TOKENS = 32768       # pb200_renoise_confidence keeps a sample's keys (4 bytes per token) in shared memory


def _confidence_tau(name: str, v) -> float:
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or v < 0:
        raise ValueError(f"{name}: the choice temperature must be a finite real number >= 0 (got {v!r})")
    return float(v)


def confidence_table(confidence_renoise, batch: int, hw: Optional[int] = None) -> Optional[torch.Tensor]:
    """``confidence_renoise`` (None, one choice temperature tau for every sample, or a list or tuple of ``batch`` entries, each
    None or tau) -> None when no sample has an entry, otherwise the CPU float32 [batch] table pb200_renoise_confidence reads:
    tau, or -1 for a sample renoised at random as add_noise does.  ValueError, before anything is enqueued, for the wrong
    length, a bool, negative or non-finite tau, and (``hw``: tokens per sample) a grid of more than MAX_CONFIDENCE_TOKENS tokens."""
    if confidence_renoise is None:
        return None
    if isinstance(confidence_renoise, (list, tuple)):
        if len(confidence_renoise) != batch:
            raise ValueError(f"confidence_renoise: got {len(confidence_renoise)} entries for a batch of {batch} (one per sample, "
                             "None for none)")
        taus = [-1.0 if v is None else _confidence_tau(f"confidence_renoise[{b}]", v) for b, v in enumerate(confidence_renoise)]
    else:
        taus = [_confidence_tau("confidence_renoise", confidence_renoise)] * batch
    if all(v < 0 for v in taus):
        return None
    if hw is not None and hw > MAX_CONFIDENCE_TOKENS:
        raise ValueError(f"confidence_renoise: a latent grid of {hw} tokens; the selection kernel takes at most "
                         f"{MAX_CONFIDENCE_TOKENS} per sample (e.g. 128 x 256)")
    return torch.tensor(taus, dtype=torch.float32)


# The notebook's sampling modes (paella_inference.ipynb cell 3).  'multinomial' draws H*W*num_labels exponentials per step; 'argmax'
# and 'quant' draw nothing.  A step with several modes sends one int32 table to the device: the mode code of every sample, then
# the samples in argmax mode, then the samples in quant mode, each list ascending.
# ------------------------------------------------------------------ token scoring
# pb200_paella_token_scores returns per token nll = lse - l_y and smooth = lse - mean_j l_j; the label-smoothed cross entropy
# torch.nn.CrossEntropyLoss(label_smoothing=eps, reduction='none') computes is (1 - eps) nll + eps smooth.
def check_label_smoothing(eps) -> float:
    """``label_smoothing`` -> the float.  ValueError unless it is a real number in [0, 1] (a bool is not one)."""
    if isinstance(eps, bool) or not isinstance(eps, (int, float)) or not 0.0 <= float(eps) <= 1.0:
        raise ValueError(f"label_smoothing: expected a number in [0, 1] (got {eps!r})")
    return float(eps)


def smoothed_loss(nll: torch.Tensor, smooth: torch.Tensor, eps: float) -> torch.Tensor:
    """(1 - eps) nll + eps smooth in the tensors' dtype; ``nll`` itself (the same tensor) at eps = 0."""
    if eps == 0.0:
        return nll
    return nll.mul(1.0 - eps).add_(smooth, alpha=eps)


def score_cfg_params(cfg, batch: int) -> Optional[torch.Tensor]:
    """``cfg`` of Paella.token_scores (None, a real number, or a CPU float tensor [batch]) -> None or the CPU params table
    float32 [batch, 3] of (cfg, 1 - cfg, 1) that sampling_params_table builds at temperature 1.  ValueError (nothing enqueued)
    for a bad value."""
    if cfg is None:
        return None
    if torch.is_tensor(cfg):
        cfgs = per_sample_values("cfg", cfg, batch)
    elif isinstance(cfg, bool) or not isinstance(cfg, (int, float)) or not math.isfinite(cfg):
        raise ValueError(f"cfg: expected None, a finite number or a CPU tensor [{batch}] (got {cfg!r})")
    else:
        cfgs = [float(cfg)] * batch
    return sampling_params(cfgs, [1.0] * batch)


def check_score_levels(levels) -> list:
    """``levels`` of utils.score -> a list of floats.  ValueError unless it is a non-empty list, tuple or 1-D CPU tensor of
    finite numbers in [0, 1] (a bool is not one)."""
    if torch.is_tensor(levels):
        if levels.device.type != "cpu" or levels.dim() != 1 or not levels.is_floating_point():
            raise ValueError(f"levels: expected a 1-D CPU floating-point tensor (got {levels.dtype} of shape {list(levels.shape)} "
                             f"on {levels.device})")
        levels = levels.tolist()
    if not isinstance(levels, (list, tuple)) or not levels:
        raise ValueError("levels: expected a non-empty sequence of noise levels in [0, 1]")
    for i, v in enumerate(levels):
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not 0.0 <= float(v) <= 1.0:
            raise ValueError(f"levels[{i}]: expected a number in [0, 1] (got {v!r})")
    return [float(v) for v in levels]


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


def renoise_confidence(x: torch.Tensor, t: torch.Tensor, tau: torch.Tensor, logp: torch.Tensor, random_x: torch.Tensor, generator=None,
                       src: Optional[torch.Tensor] = None, region: Optional[torch.Tensor] = None):
    """add_noise with the confidence rule (pb200_renoise_confidence): sample b (tau fp32 [B] on the device, >= 0) renoises its
    floor(t_b N) tokens of smallest key logp + tau t g(u), u being the uniforms add_noise draws; a sample with tau < 0 is
    add_noise's.  ``logp``: fp32, x's log-probabilities (Paella.token_logprob).  Takes exactly add_noise's draws from ``generator``
    (None, one, or a list of B).  ``random_x`` is required.  Returns (out, mask) like add_noise."""
    x = x.contiguous()
    B, hw = x.shape[0], x[0].numel()
    out, mask = torch.empty_like(x), torch.empty_like(x)
    src = src.contiguous() if src is not None else None
    args = (ptr(x), ptr(random_x.contiguous()), ptr(src), ptr(_region_u8(region)))
    rest = (ptr(logp.contiguous()), ptr(t.contiguous().float()), ptr(tau.contiguous()), B, hw)
    if per_sample(generator):
        check_generators(generator, B, x.device)
        check_per_sample_numel(hw)
        table = philox_table(generator, hw, x.device)
        check(lib().pb200_renoise_confidence_per_sample(*args, None, *rest, ptr(table), ptr(out), ptr(mask), current_stream()),
              "pb200_renoise_confidence_per_sample")
        return out, mask
    seed, off = take_philox(x.numel(), x.device, generator)
    check(lib().pb200_renoise_confidence(*args, *rest, seed, off, ptr(out), ptr(mask), current_stream()), "pb200_renoise_confidence")
    return out, mask


def renoise_confidence_per_sample(x: torch.Tensor, t: torch.Tensor, tau: torch.Tensor, logp: torch.Tensor, random_x: torch.Tensor,
                                  table: torch.Tensor, out: torch.Tensor, mask: Optional[torch.Tensor] = None,
                                  slot: Optional[torch.Tensor] = None, src: Optional[torch.Tensor] = None,
                                  region: Optional[torch.Tensor] = None) -> None:
    """add_noise_per_sample with the confidence rule of renoise_confidence, in one launch: the same (seed, offset) ``table``, slot
    map, src and region; ``logp`` fp32 by sample like x, ``tau`` fp32 [B] (< 0: add_noise_per_sample's rule)."""
    B, hw = x.shape[0], x[0].numel()
    check(lib().pb200_renoise_confidence_per_sample(ptr(x), ptr(random_x), ptr(src), ptr(_region_u8(region)), ptr(slot), ptr(logp),
                                                    ptr(t), ptr(tau), B, hw, ptr(table), ptr(out), ptr(mask), current_stream()),
          "pb200_renoise_confidence_per_sample")


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
             ln_stat=None, ln_wsum=None, ln_shift=None, ln_mean_out=None) -> torch.Tensor:
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
