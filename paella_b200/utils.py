"""The sampling loop — ``sample()`` in the reference's three signatures over one fused core.

  sample()               ref/src/utils.py:35-55
  sample_distributed()   ref/src_distributed/utils.py:97-126   (init_x, per-step cfg, sampling_conditional_steps)
  sample_notebook()      paella_inference.ipynb cell 3          (mode, attn_weights, returns intermediates; attn_weights
                                                                 may also be one vector per sample, mode and
                                                                 sampling_quant_steps one entry per sample)

Per step the reference runs two forwards, materialises 2 x [B,8192,H,W] fp32 logits and makes ~20 passes
over them.  Here: conditional and unconditional rows run as ONE batch of 2B through the denoiser (their
conditioning K/V are computed once per call, not per step), and the out_mapper GEMM, CFG mix, temperature,
softmax and multinomial draw are a single kernel.  All random draws (randint, multinomial's exponential_,
add_noise's rand_like) come from the torch CUDA generator's own Philox stream, consumed op by op like the
reference does, so ``torch.manual_seed`` means the same thing.  ``generator=[g_0, ..., g_{B-1}]`` gives each sample its own
stream, consumed in the order a batch-1 loop would: randint over H*W, then per step the multinomial's exponential_ over
H*W*num_labels (if the step draws) and add_noise's rand over H*W (if it renoises).  A sample's draws then depend only on
its own seed; its tokens too, bit for bit, where the forward is batch-invariant (DESIGN.md §3 Numerics): on the default
model with ``model.batch_invariant = True``, on the tiny test model in either mode.

Per-sample settings: ``cfg``, ``temperature``, ``t_start`` and ``t_end`` each also take a CPU float tensor whose first
dimension is B (``cfg`` [B] in ``sample``, [B, 2] in the other two; ``temperature`` [B, 2]; ``t_start`` / ``t_end`` [B]), in
any mix with scalar ones.  Sample i is then computed with exactly the scalars a call on its own settings would use: its
schedules come from the same torch.linspace calls, and the kernels see the same fp32 constants.  The [steps][B] table is
built on the host once per call and copied to the device once, so the step loop gets no host synchronisation.

Inpainting and outpainting: ``region`` (sample_distributed, sample_notebook), a bool tensor [B, H, W], True where tokens are
generated, with ``init_x`` holding the source tokens kept everywhere else.  The loop starts from where(region, randint, init_x),
puts init_x back outside the region after every step's sampling, and renoises only inside it (mask & region); its random draws
are those of the call without a region, so a generator ends at the same offset.  An all-True region is the call without
init_x, bit for bit; an all-False one returns init_x.  ``token_region`` and ``outpaint_canvas`` build the arguments from a
pixel mask or from a smaller token grid placed on a larger canvas.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import torch

from . import ops
from .modules import Paella


def _zeros_like_inputs(inputs: Dict[str, torch.Tensor]):
    return {k: (torch.zeros_like(v) if torch.is_tensor(v) else v) for k, v in inputs.items() if v is not None}


def _cfg_schedule(cfg, batch: int, steps: int):
    """``cfg`` of sample_distributed / sample_notebook -> per-step values: None, one list (scalar ``(start, end)``), or one
    list per sample (a CPU tensor [B, 2]), each from the torch.linspace call the scalar form makes."""
    if cfg is None:
        return None
    if torch.is_tensor(cfg):
        return [torch.linspace(a, b, steps).tolist() for a, b in ops.per_sample_values("cfg", cfg, batch, pair=True)]
    return torch.linspace(cfg[0], cfg[1], steps).tolist()


def sampling_schedule(batch: int, steps: int, temperature, cfgs, t_start, t_end, per_sample_cfg: bool = False,
                      always: bool = False):
    """The per-call table of per-sample settings, or None when every argument is scalar (and not ``always``).

    ``temperature``: (start, end) or a CPU tensor [B, 2]; ``t_start`` / ``t_end``: floats or CPU tensors [B]; ``cfgs``: None, the
    per-step values, or (``per_sample_cfg``) one such list per sample.  Returns CPU float32 (params [steps, B, 3] of
    (cfg, 1 - cfg, 1/T), r [steps + 1, B] of the noise levels): sample i's rows are the torch.linspace values a call on its
    settings alone uses, as the fp32 constants the kernels derive from them (ops.sampling_params).  ValueError for a bad
    per-sample value or a temperature <= 0."""
    if not (always or per_sample_cfg or any(torch.is_tensor(v) for v in (temperature, t_start, t_end))):
        return None
    if torch.is_tensor(temperature):
        tp = ops.per_sample_values("temperature", temperature, batch, pair=True)
        ops.check_temperatures("temperature", [v for pair in tp for v in pair])
        temps = torch.stack([torch.linspace(a, b, steps) for a, b in tp])
    else:
        ops.check_temperatures("temperature", temperature)
        temps = torch.linspace(temperature[0], temperature[1], steps).expand(batch, steps)
    ts = ops.per_sample_values("t_start", t_start, batch) if torch.is_tensor(t_start) else [t_start] * batch
    te = ops.per_sample_values("t_end", t_end, batch) if torch.is_tensor(t_end) else [t_end] * batch
    r = torch.stack([torch.linspace(a, b, steps + 1) for a, b in zip(ts, te)])
    if cfgs is None:
        c = [[0.0] * steps] * batch
    else:
        c = cfgs if per_sample_cfg else [list(cfgs)] * batch
    params = ops.sampling_params(c, temps.tolist())
    return params.transpose(0, 1).contiguous(), r.t().contiguous()


def check_region(region, init_x, latent_shape, device) -> None:
    """ValueError unless ``region`` is None or a bool tensor of ``latent_shape`` [B, H, W] on the CPU or on ``device``, with an
    ``init_x`` of the same shape and placement (the source tokens)."""
    if region is None:
        return
    if init_x is None:
        raise ValueError("region needs init_x: the source tokens kept outside the region")
    device = torch.device(device)
    for name, v in (("region", region), ("init_x", init_x)):
        if not torch.is_tensor(v):
            raise ValueError(f"{name}: expected a tensor (got {type(v).__name__})")
        if tuple(v.shape) != tuple(latent_shape):
            raise ValueError(f"{name} of shape {list(v.shape)}; expected {list(latent_shape)}")
        if v.device.type != "cpu" and v.device != device:
            raise ValueError(f"{name} is on {v.device}, the model on {device}")
    if region.dtype != torch.bool:
        raise ValueError(f"region: expected a bool tensor, True where tokens are generated (got {region.dtype})")
    if init_x.dtype.is_floating_point or init_x.dtype == torch.bool:
        raise ValueError(f"init_x: expected integer token indices (got {init_x.dtype})")


def token_region(pixel_mask: torch.Tensor, patch: int = 4) -> torch.Tensor:
    """The token region of a pixel mask for the f4 codec: bool [..., h, w] (True = regenerate) -> bool [..., h/4, w/4], True
    where any pixel of the token's 4x4 patch is True.  CPU tensors, no device work."""
    if not torch.is_tensor(pixel_mask) or pixel_mask.device.type != "cpu":
        raise ValueError("token_region: expected a CPU tensor")
    if pixel_mask.dim() < 2 or pixel_mask.shape[-2] % patch or pixel_mask.shape[-1] % patch:
        raise ValueError(f"token_region: a pixel mask of shape {list(pixel_mask.shape)}; its last two sizes must be multiples of {patch}")
    h, w = pixel_mask.shape[-2:]
    m = pixel_mask.bool().reshape(*pixel_mask.shape[:-2], h // patch, patch, w // patch, patch)
    return m.any(-1).any(-2)


def outpaint_canvas(tokens: torch.Tensor, canvas_hw, top: int, left: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Outpainting arguments: ``tokens`` int [B, h, w] placed with its top-left corner at (top, left) of a canvas
    ``canvas_hw`` = (H, W).  Returns (init_x int64 [B, H, W], region bool [B, H, W]): the source tokens on the canvas (0
    elsewhere) and a region that is True everywhere except under them.  CPU tensors, no device work."""
    if not torch.is_tensor(tokens) or tokens.device.type != "cpu" or tokens.dim() != 3:
        raise ValueError("outpaint_canvas: expected CPU tokens [B, h, w]")
    B, h, w = tokens.shape
    H, W = int(canvas_hw[0]), int(canvas_hw[1])
    if not (0 <= top and top + h <= H and 0 <= left and left + w <= W):
        raise ValueError(f"outpaint_canvas: a {h}x{w} grid at ({top}, {left}) does not fit a {H}x{W} canvas")
    init_x = torch.zeros(B, H, W, dtype=torch.int64)
    init_x[:, top:top + h, left:left + w] = tokens
    region = torch.ones(B, H, W, dtype=torch.bool)
    region[:, top:top + h, left:left + w] = False
    return init_x, region


def _sample_core(model: Paella, model_inputs, latent_shape, unconditional_inputs, init_x, steps, renoise_steps, temperature,
                 cfgs, t_start, t_end, sampling_conditional_steps, mode, attn_weights, exact, collect, sampling_quant_steps=None,
                 codebook=None, generator=None, per_sample_cfg=False, region=None, modes=None):
    """``modes``: None, or per step the list of B mode names (sampling_modes) -- a step whose modes differ samples each row in
    its own mode (Paella.sample_tokens_modes), a step whose modes agree takes the scalar path in that mode."""
    B, H, W = latent_shape
    dev = model._device()
    check_region(region, init_x, latent_shape, dev)
    use_cfg_any = cfgs is not None
    mixed_steps = modes is not None and any(len(set(ms)) > 1 for ms in modes)
    sched = sampling_schedule(B, steps, temperature, cfgs, t_start, t_end, per_sample_cfg, always=mixed_steps)
    w_table = None
    if isinstance(attn_weights, (list, tuple)):       # per-sample vectors, for the conditional rows only
        w_table = ops.attn_weights_table(attn_weights, B, [model.max_attn_weights((H, W), model.conditioning_seq_len(model_inputs))] * B)
    if ops.per_sample(generator):
        ops.check_generators(generator, B, dev)
        ops.check_per_sample_numel(H * W * model.num_labels)
    with torch.inference_mode():
        # one copy for the whole loop: [steps][B][3] params and [steps + 1][B] noise levels, and a CPU region
        region_host = region is not None and region.device.type == "cpu"
        parts = (list(sched) if sched is not None else []) + ([region] if region_host else [])
        parts_d = ops.to_device_packed(parts, dev) if parts else []
        if sched is not None:
            params_d, r_d = parts_d[0], parts_d[1]
        region_d = None
        if region is not None:       # bool [B, H, W], True where tokens are generated
            region_d = parts_d[-1] if region_host else region.contiguous()
        w_len = None
        if w_table is not None:      # one copy for the whole loop
            attn_weights, w_len = ops.attn_weights_to_device(*w_table, dev)
        init_noise = ops.randint(model.num_labels, (B, H, W), dev, generator)
        if region_d is not None:     # where(region, init_noise, init_x)
            src_d = init_x.to(device=dev, dtype=torch.int64).contiguous()
            neg_t = torch.full((B,), -1.0, dtype=torch.float32, device=dev)
            sampled = ops.composite(init_noise, src_d, region_d, neg_t)
        else:
            sampled = init_x.to(dev) if init_x is not None else init_noise.clone()
        if sched is None:
            t_list = torch.linspace(t_start, t_end, steps + 1)
            temperatures = torch.linspace(temperature[0], temperature[1], steps)
        groups = [model_inputs] + ([unconditional_inputs] if use_cfg_any else [])
        cond_full = model.prepare_conditioning(groups, (H, W))
        cond_only = None
        intermediates = []
        for i in range(steps):
            step_modes = None
            if modes is not None:
                step_modes = modes[i] if len(set(modes[i])) > 1 else None
                mode = modes[i][0]
            elif sampling_quant_steps is not None and i >= sampling_quant_steps:
                mode = "quant"
            guided = use_cfg_any and i < sampling_conditional_steps
            if guided:
                cond, tokens = cond_full, sampled          # one (tokens, r) per CFG pair, see Paella.features
            elif use_cfg_any:
                if cond_only is None:
                    cond_only = model.prepare_conditioning([model_inputs], (H, W))
                cond, tokens = cond_only, sampled
            else:
                cond, tokens = cond_full, sampled
            if sched is None:
                r = torch.full((tokens.shape[0],), float(t_list[i]), dtype=torch.float32, device=dev)
                cfg_i, temp_i = (float(cfgs[i]) if guided else None), float(temperatures[i])
            else:
                r, params_i = r_d[i], params_d[i]
            feats = model.features(tokens, r, cond, attn_weights, B if attn_weights is not None else 0, cfg_pairs=guided, w_len=w_len)
            if step_modes is not None:
                sampled = _sample_modes_step(model, feats, B, H, W, guided, params_i, step_modes, generator, codebook, dev)
            elif mode == "multinomial" and not exact:
                if sched is None:
                    sampled = model.sample_tokens(feats, B, H, W, cfg_i, temp_i, generator)
                else:
                    sampled = model.sample_tokens_params(feats, B, H, W, guided, params_i, generator)
            else:
                n = B * H * W
                lc = model.logits_from_features(feats[:n], B, H, W)
                lu = model.logits_from_features(feats[n:], B, H, W) if guided else None
                if mode == "quant":
                    if codebook is None:
                        raise ValueError("mode='quant' needs the VQGAN codebook: pass vqmodel=... (the notebook uses its global `vqmodel`)")
                    if sched is None:
                        sampled = ops.resample_quant(lc, lu, cfg_i if guided else 0.0, temp_i, codebook)
                    else:
                        sampled = ops.resample_quant_params(lc, lu, params_i, codebook)
                elif sched is None:
                    sampled = ops.resample_logits(lc, lu, cfg_i if guided else 0.0, temp_i, mode, generator)
                else:
                    sampled = ops.resample_logits_params(lc, lu, params_i, mode, generator)
            # outside the region the tokens are init_x's again; a renoising step composites in its own launch, so the
            # composite is a launch of its own only where an intermediate shows it or nothing renoises
            if region_d is not None and (collect or i >= renoise_steps):
                sampled = ops.composite(sampled, src_d, region_d, neg_t)
            if collect:
                intermediates.append(sampled)
            if i < renoise_steps:
                if sched is None:
                    t_next = torch.full((B,), float(t_list[i + 1]), dtype=torch.float32, device=dev)
                else:
                    t_next = r_d[i + 1]
                if region_d is None:
                    sampled = model.add_noise(sampled, t_next, random_x=init_noise, generator=generator)[0]
                else:
                    sampled = model.add_noise(sampled, t_next, random_x=init_noise, generator=generator, src=src_d, region=region_d)[0]
                if collect:
                    intermediates.append(sampled)
    return sampled, intermediates


def _sample_modes_step(model, feats, B, H, W, guided, params, step_modes, generators, codebook, dev):
    """One step of a batch whose samples are in different modes, on per-sample generators: the multinomial samples draw what
    a batch-1 step draws on their own generators, the others draw nothing.  The draws and the mode table go to the device in
    one asynchronous copy."""
    vals = []
    for g, md in zip(generators, step_modes):
        vals += ops.philox_values([g], H * W * model.num_labels, dev) if md == "multinomial" else [0, 0]
    seed_d, table_d = ops.to_device_packed([torch.tensor(vals, dtype=torch.int64).view(-1, 2), ops.mode_table(step_modes)], dev)
    return model.sample_tokens_modes(feats, B, B if guided else 0, H, W, params, seed_d, step_modes, table_d, codebook)


def sampling_modes(mode, sampling_quant_steps, batch: int, steps: int, generator=None, exact: bool = False, codebook=None):
    """sample_notebook's ``mode`` and ``sampling_quant_steps`` -> None when both are scalar or a list's entries are all equal
    (the scalar path), otherwise per step the list of ``batch`` mode names (ops.mode_at).  ValueError, before anything is
    enqueued, for a list of the wrong length, an unknown mode, a quant step that is not None or an int >= 0, 'quant' at some
    step without a codebook, and -- for a step whose modes differ -- a call without per-sample generators or with exact=True."""
    if not isinstance(mode, (list, tuple)) and not isinstance(sampling_quant_steps, (list, tuple)):
        return None
    per = []
    for name, v in (("mode", mode), ("sampling_quant_steps", sampling_quant_steps)):
        if isinstance(v, (list, tuple)):
            if len(v) != batch:
                raise ValueError(f"{name}: got {len(v)} entries for a batch of {batch} (one per sample)")
            per.append(list(v))
        else:
            per.append([v] * batch)
    ms = [ops.check_mode(f"mode[{b}]", v) for b, v in enumerate(per[0])]
    qs = [ops.check_quant_steps(f"sampling_quant_steps[{b}]", v) for b, v in enumerate(per[1])]
    table = [[ops.mode_at(md, q, i) for md, q in zip(ms, qs)] for i in range(steps)]
    if codebook is None and any("quant" in row for row in table):
        raise ValueError("mode='quant' needs the VQGAN codebook: pass vqmodel=... (the notebook uses its global `vqmodel`)")
    if len(set(ms)) == 1 and len(set(qs)) == 1:
        return None
    if any(len(set(row)) > 1 for row in table):
        if not ops.per_sample(generator):
            raise ValueError("samples in different sampling modes draw per sample: pass generator=[g_0, ..., g_{B-1}]")
        if exact:
            raise ValueError("exact=True is the multinomial parity path; it does not take per-sample modes")
    return table


def load_conditional_models(byt5_model_name, vqgan_path, device):
    """ref/src/utils.py:24-32: the f4 codec from ``vqgan_path`` (a ``{'state_dict': ...}`` checkpoint, as saved by the
    reference's training code) and the ByT5 text encoder.  The codec is this package's VQModel; the text encoder is
    the third-party ``transformers`` model exactly as in the reference (outside the hot path, SURVEY.md §8f.4) —
    ``byt5_model_name=None`` skips it."""
    from .vqgan import VQModel
    vqgan = VQModel().to(device)
    ckpt = torch.load(vqgan_path, map_location=device)
    vqgan.load_state_dict(ckpt["state_dict"] if isinstance(ckpt, dict) and "state_dict" in ckpt else ckpt)
    vqgan.eval().requires_grad_(False)
    if byt5_model_name is None:
        return vqgan, None
    from transformers import AutoTokenizer, T5EncoderModel
    byt5 = T5EncoderModel.from_pretrained(byt5_model_name).to(device).eval().requires_grad_(False)
    byt5_tokenizer = AutoTokenizer.from_pretrained(byt5_model_name)
    return vqgan, (byt5_tokenizer, byt5)


def _decode_tail(tokens, decode, decode_output):
    """The step after the path (SURVEY.md §8 f2; ref/src_distributed/train.py:168-171, notebook nb:354-357): the final token
    grid goes straight into the f4 decoder on the same stream -- no host round trip, no separate clamp / byte pass."""
    if decode is None:
        return tokens
    if decode_output == "uint8":
        return decode.decode_indices_u8(tokens)
    if decode_output == "clamp":
        return decode.decode_indices_clamped(tokens)
    if decode_output == "raw":
        return decode.decode_indices(tokens)
    raise ValueError(f"decode_output={decode_output!r}: expected 'uint8', 'clamp' or 'raw'")


def sample(model, model_inputs, latent_shape, unconditional_inputs=None, steps=12, renoise_steps=11, temperature=(1.0, 0.2),
           cfg=8.0, t_start=1.0, t_end=0.0, device="cuda", exact=False, decode=None, decode_output="uint8", generator=None):
    """ref/src/utils.py:35-55 (same positional/keyword arguments; ``device`` is accepted and must be the model's).
    ``exact=True`` materialises the logits and uses the op-for-op torch arithmetic (parity path).
    ``decode=vqmodel`` appends the reference callers' next step, ``vqmodel.decode_indices(tokens).clamp(0, 1)``, fused on the
    tail: returns uint8 NHWC images (``decode_output='uint8'``), clamped fp32 NCHW ('clamp') or unclamped fp32 NCHW ('raw').
    ``generator``: None draws on the default CUDA generator; one CUDA ``torch.Generator`` replaces it; a list of B of them gives
    every sample its own stream -- row i draws what this call with batch 1 on sample i's inputs draws after
    ``torch.manual_seed(generator[i].initial_seed())`` (and equals it where the forward is batch-invariant, DESIGN.md §3),
    and leaves generator i where that call leaves the default generator.
    Per-sample settings (module docstring): ``cfg`` [B], ``temperature`` [B, 2], ``t_start`` / ``t_end`` [B].  A per-sample cfg
    of 0 is unguided like the scalar ``cfg=0``; so is 1.0, and an all-zero tensor makes the whole call unguided."""
    per_sample_cfg = torch.is_tensor(cfg)
    if per_sample_cfg:
        cfg_vals = [v if v else 1.0 for v in ops.per_sample_values("cfg", cfg, latent_shape[0])]   # f*1 + u*0 = f
        cfgs = [[v] * steps for v in cfg_vals] if any(cfg.tolist()) else None
        per_sample_cfg = cfgs is not None
    else:
        cfgs = [cfg] * steps if cfg else None
    if cfgs is not None and unconditional_inputs is None:
        raise TypeError("sample(): cfg is set but unconditional_inputs is None")
    out, _ = _sample_core(model, model_inputs, tuple(latent_shape), unconditional_inputs, None, steps, renoise_steps,
                          temperature, cfgs, t_start, t_end, steps, "multinomial", None, exact, False, generator=generator,
                          per_sample_cfg=per_sample_cfg)
    return _decode_tail(out, decode, decode_output)


def sample_distributed(model, model_inputs, unconditional_inputs, latent_shape, init_x=None, steps=12, renoise_steps=None,
                       temperature=(0.7, 0.3), cfg=(8.0, 8.0), t_start=1.0, t_end=0.0, sampling_conditional_steps=None,
                       exact=False, generator=None, region=None):
    """ref/src_distributed/utils.py:97-126.  ``generator`` as in ``sample``: a shard given ``generators[lo:hi]`` draws what
    rows [lo, hi) of the single-GPU call draw.  Per-sample settings (module docstring): ``cfg`` and ``temperature`` [B, 2],
    ``t_start`` / ``t_end`` [B]; a shard given ``settings[lo:hi]`` computes what rows [lo, hi) compute.  ``region`` (module
    docstring): bool [B, H, W] on the CPU or the model's device, True where tokens are generated; ``init_x`` then holds the
    tokens kept elsewhere.  ValueError, before anything is enqueued and before any generator advances, for a region without
    init_x, of another shape or dtype, or on another device."""
    if sampling_conditional_steps is None:
        sampling_conditional_steps = steps
    if renoise_steps is None:
        renoise_steps = steps - 1
    cfgs = _cfg_schedule(cfg, latent_shape[0], steps)
    out, _ = _sample_core(model, model_inputs, tuple(latent_shape), unconditional_inputs, init_x, steps, renoise_steps,
                          temperature, cfgs, t_start, t_end, sampling_conditional_steps, "multinomial", None, exact, False,
                          generator=generator, per_sample_cfg=torch.is_tensor(cfg), region=region)
    return out


def sample_notebook(model, model_inputs, latent_shape, unconditional_inputs=None, init_x=None, steps=12, renoise_steps=None,
                    temperature=(0.7, 0.3), cfg=(8.0, 8.0), mode='multinomial', t_start=1.0, t_end=0.0,
                    sampling_conditional_steps=None, sampling_quant_steps=None, attn_weights=None, exact=False, vqmodel=None,
                    generator=None, region=None):
    """paella_inference.ipynb cell 3: returns (sampled, intermediate_images).  ``vqmodel`` replaces the notebook's global
    of the same name for ``mode='quant'`` / ``sampling_quant_steps`` (softmax @ codebook -> nearest code).  ``generator`` as
    in ``sample``; per-sample settings as in ``sample_distributed``.  ``attn_weights``: one 1-D tensor for every sample, or a
    list or tuple of B entries, each None or a 1-D CPU float tensor that weights sample b's conditional forward alone (the
    unconditional rows are never weighted, as in the notebook).  Row i then equals row i of the call with vector i for every
    sample.  ValueError, before anything is enqueued and before any generator advances, for the wrong number of entries, a
    CUDA, non-1-D or non-finite tensor, or a vector longer than the smallest key count the sample sees in an AttnBlock.
    ``region`` as in ``sample_distributed``; every intermediate holds init_x's tokens outside it.
    Per-sample modes: ``mode`` may be a list or tuple of B mode names and ``sampling_quant_steps`` one of B entries, each None
    or an int >= 0; row i then equals row i of the call with mode i and quant step i for every sample, on per-sample
    generators.  A call whose modes differ within a step needs ``generator=[g_0, ..., g_{B-1}]`` (the argmax and quant rows draw
    nothing, the multinomial ones draw per sample); one whose entries are all equal is the scalar call (sampling_modes)."""
    if sampling_conditional_steps is None:
        sampling_conditional_steps = steps
    if renoise_steps is None:
        renoise_steps = steps - 1
    if unconditional_inputs is None:
        unconditional_inputs = _zeros_like_inputs(model_inputs)
    cfgs = _cfg_schedule(cfg, latent_shape[0], steps)
    codebook = vqmodel.vquantizer.codebook.weight.data if vqmodel is not None else None
    modes = sampling_modes(mode, sampling_quant_steps, latent_shape[0], steps, generator, exact, codebook)
    if modes is None and isinstance(mode, (list, tuple)):
        mode = mode[0]
    if modes is None and isinstance(sampling_quant_steps, (list, tuple)):
        sampling_quant_steps = sampling_quant_steps[0]
    return _sample_core(model, model_inputs, tuple(latent_shape), unconditional_inputs, init_x, steps, renoise_steps,
                        temperature, cfgs, t_start, t_end, sampling_conditional_steps, mode, attn_weights, exact, True,
                        sampling_quant_steps, codebook, generator, per_sample_cfg=torch.is_tensor(cfg), region=region, modes=modes)
