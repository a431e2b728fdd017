"""The sampling loop — ``sample()`` in the reference's three signatures over one fused core.

  sample()               ref/src/utils.py:35-55
  sample_distributed()   ref/src_distributed/utils.py:97-126   (init_x, per-step cfg, sampling_conditional_steps)
  sample_notebook()      paella_inference.ipynb cell 3          (mode, attn_weights, returns intermediates)

Per step the reference runs two forwards, materialises 2 x [B,8192,H,W] fp32 logits and makes ~20 passes
over them.  Here: conditional and unconditional rows run as ONE batch of 2B through the denoiser (their
conditioning K/V are computed once per call, not per step), and the out_mapper GEMM, CFG mix, temperature,
softmax and multinomial draw are a single kernel.  All random draws (randint, multinomial's exponential_,
add_noise's rand_like) come from the torch CUDA generator's own Philox stream, consumed op by op like the
reference does, so ``torch.manual_seed`` means the same thing.  ``generator=[g_0, ..., g_{B-1}]`` gives each sample its own
stream, consumed in the order a batch-1 loop would: randint over H*W, then per step the multinomial's exponential_ over
H*W*num_labels (if the step draws) and add_noise's rand over H*W (if it renoises).  A sample's draws then depend only on
its own seed; its tokens too, bit for bit, where the forward is batch-invariant (DESIGN.md §3 Numerics).
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import torch

from . import ops
from .modules import Paella


def _zeros_like_inputs(inputs: Dict[str, torch.Tensor]):
    return {k: (torch.zeros_like(v) if torch.is_tensor(v) else v) for k, v in inputs.items() if v is not None}


def _sample_core(model: Paella, model_inputs, latent_shape, unconditional_inputs, init_x, steps, renoise_steps, temperature,
                 cfgs, t_start, t_end, sampling_conditional_steps, mode, attn_weights, exact, collect, sampling_quant_steps=None,
                 codebook=None, generator=None):
    B, H, W = latent_shape
    dev = model._device()
    use_cfg_any = cfgs is not None
    if ops.per_sample(generator):
        ops.check_generators(generator, B, dev)
        ops.check_per_sample_numel(H * W * model.num_labels)
    with torch.inference_mode():
        init_noise = ops.randint(model.num_labels, (B, H, W), dev, generator)
        sampled = init_x.to(dev) if init_x is not None else init_noise.clone()
        t_list = torch.linspace(t_start, t_end, steps + 1)
        temperatures = torch.linspace(temperature[0], temperature[1], steps)
        groups = [model_inputs] + ([unconditional_inputs] if use_cfg_any else [])
        cond_full = model.prepare_conditioning(groups, (H, W))
        cond_only = None
        intermediates = []
        for i in range(steps):
            if sampling_quant_steps is not None and i >= sampling_quant_steps:
                mode = "quant"
            guided = use_cfg_any and i < sampling_conditional_steps
            t = float(t_list[i])
            if guided:
                cond, tokens = cond_full, sampled          # one (tokens, r) per CFG pair, see Paella.features
            elif use_cfg_any:
                if cond_only is None:
                    cond_only = model.prepare_conditioning([model_inputs], (H, W))
                cond, tokens = cond_only, sampled
            else:
                cond, tokens = cond_full, sampled
            r = torch.full((tokens.shape[0],), t, dtype=torch.float32, device=dev)
            feats = model.features(tokens, r, cond, attn_weights, B if attn_weights is not None else 0, cfg_pairs=guided)
            cfg_i = float(cfgs[i]) if guided else None
            if mode == "multinomial" and not exact:
                sampled = model.sample_tokens(feats, B, H, W, cfg_i, float(temperatures[i]), generator)
            else:
                n = B * H * W
                lc = model.logits_from_features(feats[:n], B, H, W)
                lu = model.logits_from_features(feats[n:], B, H, W) if guided else None
                if mode == "quant":
                    if codebook is None:
                        raise ValueError("mode='quant' needs the VQGAN codebook: pass vqmodel=... (the notebook uses its global `vqmodel`)")
                    sampled = ops.resample_quant(lc, lu, cfg_i if guided else 0.0, float(temperatures[i]), codebook)
                else:
                    sampled = ops.resample_logits(lc, lu, cfg_i if guided else 0.0, float(temperatures[i]), mode, generator)
            if collect:
                intermediates.append(sampled)
            if i < renoise_steps:
                t_next = torch.full((B,), float(t_list[i + 1]), dtype=torch.float32, device=dev)
                sampled = model.add_noise(sampled, t_next, random_x=init_noise, generator=generator)[0]
                if collect:
                    intermediates.append(sampled)
    return sampled, intermediates


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
    and leaves generator i where that call leaves the default generator."""
    cfgs = [cfg] * steps if cfg else None
    if cfgs is not None and unconditional_inputs is None:
        raise TypeError("sample(): cfg is set but unconditional_inputs is None")
    out, _ = _sample_core(model, model_inputs, tuple(latent_shape), unconditional_inputs, None, steps, renoise_steps,
                          temperature, cfgs, t_start, t_end, steps, "multinomial", None, exact, False, generator=generator)
    return _decode_tail(out, decode, decode_output)


def sample_distributed(model, model_inputs, unconditional_inputs, latent_shape, init_x=None, steps=12, renoise_steps=None,
                       temperature=(0.7, 0.3), cfg=(8.0, 8.0), t_start=1.0, t_end=0.0, sampling_conditional_steps=None,
                       exact=False, generator=None):
    """ref/src_distributed/utils.py:97-126.  ``generator`` as in ``sample``: a shard given ``generators[lo:hi]`` draws what
    rows [lo, hi) of the single-GPU call draw."""
    if sampling_conditional_steps is None:
        sampling_conditional_steps = steps
    if renoise_steps is None:
        renoise_steps = steps - 1
    cfgs = torch.linspace(cfg[0], cfg[1], steps).tolist() if cfg is not None else None
    out, _ = _sample_core(model, model_inputs, tuple(latent_shape), unconditional_inputs, init_x, steps, renoise_steps,
                          temperature, cfgs, t_start, t_end, sampling_conditional_steps, "multinomial", None, exact, False,
                          generator=generator)
    return out


def sample_notebook(model, model_inputs, latent_shape, unconditional_inputs=None, init_x=None, steps=12, renoise_steps=None,
                    temperature=(0.7, 0.3), cfg=(8.0, 8.0), mode='multinomial', t_start=1.0, t_end=0.0,
                    sampling_conditional_steps=None, sampling_quant_steps=None, attn_weights=None, exact=False, vqmodel=None,
                    generator=None):
    """paella_inference.ipynb cell 3: returns (sampled, intermediate_images).  ``vqmodel`` replaces the notebook's global
    of the same name for ``mode='quant'`` / ``sampling_quant_steps`` (softmax @ codebook -> nearest code).  ``generator`` as
    in ``sample``."""
    if sampling_conditional_steps is None:
        sampling_conditional_steps = steps
    if renoise_steps is None:
        renoise_steps = steps - 1
    if unconditional_inputs is None:
        unconditional_inputs = _zeros_like_inputs(model_inputs)
    cfgs = torch.linspace(cfg[0], cfg[1], steps).tolist() if cfg is not None else None
    codebook = vqmodel.vquantizer.codebook.weight.data if vqmodel is not None else None
    return _sample_core(model, model_inputs, tuple(latent_shape), unconditional_inputs, init_x, steps, renoise_steps,
                        temperature, cfgs, t_start, t_end, sampling_conditional_steps, mode, attn_weights, exact, True,
                        sampling_quant_steps, codebook, generator)
