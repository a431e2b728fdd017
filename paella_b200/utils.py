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

Truncated sampling: ``top_k`` and ``top_p`` (all three functions; None, a scalar, or a CPU tensor [B]) restrict each token's
multinomial draw to its k most likely codes, then to the smallest top set of them holding a fraction p of the probability
(ops.truncation_table; pb200_paella_sample_tokens_params_trunc).  The draw uses the same random numbers as without
truncation, so every generator ends at the same offset and the per-sample guarantees above hold for truncated rows too.
Argmax and quant steps are not truncated; ``exact=True`` does not take truncation.

Seamless tiling: ``tiling`` (all three functions; None / 'none', 'x', 'y' or 'xy', one for the call or a list or tuple of B values)
makes sample i's token grid wrap around on its axes: 'x' joins the left and right edges (a horizontal panorama), 'xy' all four (a
texture that repeats without a seam).  The denoiser's ResBlock depthwise convolutions then pad circularly (ops.tiling_table;
pb200_paella_features_tiled), the only place a Paella token grid meets its edges.  Tiling draws no random numbers, so every
generator ends at the same offset, and the per-sample guarantees above hold for tiled rows too.  ``sample(..., decode=vqmodel)``
decodes each image with its own tiling.

Regional prompts: ``prompt_regions`` (all three functions; None, or a list or tuple of B entries, each None or a list of at most 7
(inputs, region) pairs) gives sample i further prompts, each on a region of its token grid: ``inputs`` is a batch-1 conditioning
dict like ``model_inputs`` and ``region`` a bool [H, W] tensor (``token_region`` makes one from a pixel mask).  In the conditional
forward, every AttnBlock position attends to all self keys and, in one softmax, to the conditioning of each region its footprint
(patch_size * 2^level tokens square) touches, and to the sample's own ``model_inputs`` row where it touches no region; regions may
overlap or leave tokens uncovered.  The unconditional forward is unchanged, so negative prompts stay global.  Regional prompts draw
no random numbers, so every generator ends at the same offset, and the per-sample guarantees above hold for regional rows too
(ops.regional_table; pb200_paella_features_regional).  ValueError, before anything is enqueued and before any generator advances,
for a bad entry and for regions on a sample that also has ``attn_weights``.

Guidance prompts: ``guidance_prompts`` (all three functions; None, or a list or tuple of B entries, each None or a list of at most 7
(inputs, weight) pairs) gives sample i further global prompts in its guided mix: ``inputs`` is a batch-1 conditioning dict like
``model_inputs`` and ``weight`` a finite real number, negative for a further negative prompt.  On a guided step with scale cfg_i the
sample's logits are l_u + cfg_i * [(l_c - l_u) + sum_j w_j (l_j - l_u)], l_j being the conditional forward under term j's inputs:
one more denoiser row per term, which shares the conditioning-free prefix with its sample (pb200_paella_features_tail).  The
coefficients cfg_i, 1 - cfg_i (1 + sum w) and cfg_i w_j are computed in double from the step's torch.linspace cfg and rounded to fp32;
they sum to 1, so the mix runs on the features before the out_mapper GEMM (pb200_paella_guidance_mix), and the sample is then drawn
from the mixed row as an unguided one.  Terms act on guided steps only and draw no random numbers, so every generator ends at the
same offset, and the per-sample guarantees above hold for such rows too.  Term prompts are global: regional prompts and
``attn_weights`` apply to the sample's conditional row only.  Argmax and quant steps, truncation, tiling and regions see the mixed
row.  ValueError, before anything is enqueued and before any generator advances, for the wrong number of entries, more than 7
terms, bad inputs or a non-finite weight, terms in a call that is not guided (cfg None; in ``sample`` a cfg of 0, or a per-sample
cfg of 0 on a sample with terms), and terms with ``exact=True``.

Attention maps: ``attention_maps=True`` (all three functions) also returns maps, float32 [B, S, H, W] on the model's device: for
key s of sample i's conditioning sequence (gen_c_embeddings order: the byt5 rows, then clip_seq_len rows per clip and per clip_image
embedding) and token (y, x), the mean over the call's steps, every AttnBlock and its heads of the post-softmax, post-attn_weights
probability that the block position holding the token gives the key, as the reference's CustomMultiheadAttention returns it with
need_weights=True (pb200_paella_features_maps).  Only the sample's own conditional row contributes, on every step, guided or not.
Maps draw no random numbers and change no token: tokens, intermediates and generator offsets are those of the call without them,
and a sample's maps depend only on its own request where the forward is batch-invariant.  ValueError, before anything is enqueued
and before any generator advances, for a flag that is not a bool and for maps together with ``prompt_regions``.

Prompt-to-prompt editing: ``attention_source`` (all three functions; None, or a list or tuple of B entries, each None or an (a, k)
pair of ints) makes sample i an edit of sample a of the same call: on steps s < k, sample i's conditional forward (guided or not)
attends in every AttnBlock and head with sample a's attention probabilities, the joint softmax over self and conditioning keys of
a's own queries and keys in that forward, times sample i's own ``attn_weights``, applied to sample i's own values.  Run an edit from
its source's noise, by giving it its own generator seeded like the source's (``generator=[g_0, ..., g_{B-1}]``); the call does not
check it.  With the same prompt and seed an edit returns its source's tokens for any k; with another prompt it keeps the
source's layout for the first k steps (Hertz et al. 2022, "Prompt-to-Prompt Image Editing with Cross Attention Control"), and an
edit with the source's prompt and its own ``attn_weights`` is their attention re-weighting.  Unconditional rows, guidance-prompt
term rows, the source's own row and every step s >= k are never injected.  Injection draws no random numbers, so every generator
ends at the same offset, and rows that are not edits, the sources among them, are those of the call without it, bit for bit.  A
source and its edits must sit in the same shard; indices are relative to the call.  ValueError, before anything is enqueued and
before any generator advances, for the wrong length, a bad entry (a bool is not an int), a source out of range or equal to its
sample, a source that is itself injected, k outside [0, steps], ``prompt_regions`` on an edit or its source, and ``exact=True``
(ops.attention_source_table; pb200_paella_features_inject).

LoRA adapters: ``lora`` (all three functions and ``score``; None, an adapter or (adapter, scale) for every sample, or a list or tuple
of B entries, each None, an adapter or (adapter, scale)) runs sample i under its own fine-tuned adapter (paella_b200.lora.load_lora):
sample i is the reference model with W + scale * (alpha / r) * B A on the adapter's targets, the in_proj, out_proj and kv_mapper of
every AttnBlock, in every forward it takes part in -- its conditional, unconditional and guidance-prompt rows and the projections of
its own, unconditional, regional and term prompts (an adapter is part of the model, not of the prompt).  Samples on different
adapters share one denoiser batch: each row's delta comes from a segmented shrink + expand kernel after the shared GEMM
(pb200_paella_features_lora).  Adapters draw no random numbers, so every generator ends at the same offset and the per-sample
guarantees above hold for adapted rows too; rows without an adapter, or at scale 0, are those of the call without it, bit for bit.
ValueError, before anything is enqueued and before any generator advances, for the wrong length, a bad entry or non-finite scale, and
an adapter loaded for another configuration or on another device (ops.lora_table).

Perturbed-attention guidance: ``pag`` (all three functions; None, or a list or tuple of B entries, each None, a scale s or an (s,
blocks) pair) guides sample i away from its perturbed forward (Ahn et al. 2024, "Self-Rectifying Diffusion Sampling with
Perturbed-Attention Guidance"): its conditional forward in which, in every AttnBlock listed in ``blocks`` (indices in plan order,
paella_b200.lora.attn_blocks; default: the deepest level's, down and up, Paella.pag_default_blocks), each query's attention mass on the
image's own tokens goes to its own value, while its probabilities on the prompt stay as they are.  On a step s <
sampling_conditional_steps a guided sample's logits are l_u + cfg * [(l_c - l_u) + sum_j w_j (l_j - l_u)] + s (l_c - l_p), an
unguided one's (cfg None, or a per-sample cfg of 1.0) l_c + s (l_c - l_p); later steps have no perturbed row.  The perturbed forward is
one more tail row after the term rows, which reads its sample's own conditioning slot, wrap byte, adapter and ``attn_weights``
(pb200_paella_features_pag), and its coefficients join the guided mix as guidance prompts' do.  The default blocks follow PAG's choice
of the mid-block by analogy; their effect on images is unmeasured here (there are no trained weights).  PAG draws no random numbers,
so every generator ends at the same offset and the per-sample guarantees above hold; a sample with no entry or s = 0 gets the tokens
of the call without it, bit for bit.  ValueError, before anything is enqueued and before any generator advances, for the wrong length,
a non-finite or bool scale, empty, duplicated, non-int or out-of-range blocks, PAG on a sample with ``prompt_regions`` or on a
prompt-to-prompt edit or source, and ``exact=True`` (ops.pag_table).

Confidence-guided renoising: ``confidence_renoise`` (all three functions; None, one choice temperature tau for every sample, or a
list or tuple of B entries, each None or tau, a finite float >= 0) renoises sample i's least likely tokens instead of a random set,
as MaskGIT and Muse do (Chang et al. 2022, "MaskGIT", section 3.2).  On every renoising step s < renoise_steps a sample with an
entry is renoised as follows, x being the step's drawn token grid:
  1. confidence: c_j = log_softmax(l * (1/T_s))[x_j] per token, l the out_mapper product of the same fp16 operand the step's
     sampler consumed (CFG pre-mixed; guidance prompts and PAG mixed in place), T_s the sample's temperature at the step, the
     product rounded once.  It is computed so whatever drew the tokens (multinomial, argmax, quant, truncated), always under the
     untruncated tempered distribution (Paella.token_logprob; pb200_paella_token_logprob).
  2. count: n = floor(t * N) in fp32, t = t_{s+1} the sample's next noise level (the level add_noise renoises to) and N = H*W, or
     the number of tokens in the sample's ``region`` when inpainting.
  3. key: k_j = c_j + (tau * t) * g_j in fp32, g_j = -logf(-logf(u_j)), u_j exactly the uniform add_noise would draw for token j:
     same generator, same offset, same Philox element, so the generator's draws and final offset are unchanged.  A u of 0 gives
     g = -inf; a NaN key ranks lowest (renoised first).
  4. renoise: the n tokens with the smallest keys are renoised, ties broken by ascending token index; a renoised token becomes the
     initial noise's code, as with add_noise.  Tokens outside a ``region`` are never candidates and stay init_x's.
With the default schedule t_{s+1} = 1 - (s+1)/steps, tau * t is MaskGIT's annealed choice temperature tau (1 - ratio).  Samples
without an entry are, bit for bit, those of the call without the argument, and a call with no entries launches exactly what it
launches without it.  No extra random numbers are drawn, so every generator ends at the same offset and the per-sample guarantees
above hold for confidence rows too.  A call with an entry takes the per-sample table path.  ValueError, before anything is enqueued
and before any generator advances, for the wrong length, a bool, negative or non-finite tau, ``exact=True``, and a latent grid of more
than 32768 tokens (the selection kernel keeps a sample's keys in shared memory; ops.confidence_table, pb200_renoise_confidence).  Its
effect on image quality is not measured here (there are no trained weights).

Scoring: ``score`` asks the denoiser how likely a given token grid is under a prompt -- held-out evaluation of a checkpoint with
train.py's objective, reranking of candidates, or picking the prompt that best explains an image.  It noises the tokens at each
of a list of noise levels, as add_noise does, and scores each noised grid against the clean tokens with Paella.token_scores
(pb200_paella_token_scores), whose fused kernel never writes the logits.
"""
from __future__ import annotations

from collections import namedtuple
from typing import Dict, Optional, Sequence, Tuple

import torch

from . import ops
from .modules import ConditioningCache, Paella


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
                 codebook=None, generator=None, per_sample_cfg=False, region=None, modes=None, top_k=None, top_p=None, tiling=None,
                 prompt_regions=None, guidance_prompts=None, attention_maps=False, attention_source=None, lora=None, pag=None,
                 confidence_renoise=None):
    """Returns (tokens, intermediates, maps or None).  ``modes``: None, or per step the list of B mode names (sampling_modes) --
    a step whose modes differ samples each row in its own mode (Paella.sample_tokens_modes), a step whose modes agree takes the
    scalar path in that mode.  ``top_k`` / ``top_p``: the truncation of the multinomial draws (module docstring); a truncating
    call takes the per-sample table path, and so does a call with ``guidance_prompts`` (module docstring).  ``attention_maps``:
    the maps of the conditional rows (module docstring).  ``attention_source``: prompt-to-prompt injection (module docstring);
    step i passes row i of the table to the denoiser, or nothing when no sample is injected there.  ``lora``: per-sample LoRA
    adapters (module docstring).  ``pag``: perturbed-attention guidance (module docstring): on steps i < sampling_conditional_steps
    each perturbed sample has one more tail row, after the term rows, and joins the composed samples of the guided mix.
    ``confidence_renoise``: confidence-guided renoising (module docstring): each renoising step scores the drawn tokens on the
    step's own sampler operand and renoises with pb200_renoise_confidence in place of add_noise."""
    B, H, W = latent_shape
    dev = model._device()
    attention_maps = ops.check_attention_maps(attention_maps, prompt_regions)
    check_region(region, init_x, latent_shape, dev)
    trunc = ops.truncation_table(top_k, top_p, B, model.num_labels)
    wrap = ops.tiling_table(tiling, B)
    regions = ops.regional_table(prompt_regions, B, (H, W), dev)
    ops.check_regions_unweighted(regions, attn_weights)
    terms = ops.guidance_table(guidance_prompts, B)
    inj = ops.attention_source_table(attention_source, B, steps, regions, exact)
    inj_steps = [bool((row >= 0).any()) for row in inj] if inj is not None else [False] * steps
    pag_t = ops.pag_table(pag, B, model.n_attn_blocks, model.pag_default_blocks(), regions, inj, exact) if pag is not None else None
    lora_t = ops.lora_table(lora, B, model)
    entries = ops.lora_entries(lora_t, B)
    extra = [g for own in regions[1] for g in own] if regions is not None else []
    extra_lora = [entries[b] for b, own in enumerate(regions[1]) for _ in own] if regions is not None else []
    if exact and trunc is not None:
        raise ValueError("exact=True restates the reference op for op, which has no top_k / top_p truncation")
    conf = ops.confidence_table(confidence_renoise, B, H * W)
    if exact and conf is not None:
        raise ValueError("exact=True restates the reference op for op, which has no confidence-guided renoising")
    use_cfg_any = cfgs is not None
    if terms is not None and exact:
        raise ValueError("exact=True restates the reference op for op, which has no guidance prompts")
    if terms is not None and not use_cfg_any:
        raise ValueError("guidance_prompts need a guided call (cfg is None or 0)")
    mixed_steps = modes is not None and any(len(set(ms)) > 1 for ms in modes)
    sched = sampling_schedule(B, steps, temperature, cfgs, t_start, t_end, per_sample_cfg,
                              always=mixed_steps or trunc is not None or terms is not None or pag_t is not None or conf is not None)
    mix = None
    pag_src = []
    n_mix = min(steps, sampling_conditional_steps)
    if terms is not None or pag_t is not None:
        # the composed samples' mix table over the guided steps; their params rows there become (1, 0, 1/T): f*1 + u*0 = f.  The
        # batch is [B conditional; B unconditional (guided calls); term rows by sample, then term; perturbed rows by sample]
        tl = terms if terms is not None else [[] for _ in range(B)]
        pag_s = pag_t[0] if pag_t is not None else [0.0] * B
        comp = [b for b in range(B) if tl[b] or pag_s[b] != 0.0]
        n_reg = len(extra)
        term_src, term_rows, k = [], [], 2 * B if use_cfg_any else B
        for b in comp:
            term_rows.append(list(range(k, k + len(tl[b]))))
            term_src += [b] * len(tl[b])
            k += len(tl[b])
        pag_src = [b for b in comp if pag_s[b] != 0.0]
        pag_row = {b: k + j for j, b in enumerate(pag_src)}
        extra = extra + [inputs for b in comp for inputs, _ in tl[b]]
        extra_lora = extra_lora + [entries[b] for b in comp for _ in tl[b]]
        step_cfgs = [[(cfgs[b] if per_sample_cfg else cfgs)[i] if use_cfg_any else None for b in comp] for i in range(n_mix)]
        mix_rows, mix_coef = ops.guidance_mix_table([[w for _, w in tl[b]] for b in comp], comp,
                                                    [B + b for b in comp] if use_cfg_any else None, term_rows, step_cfgs,
                                                    [pag_s[b] for b in comp], [pag_row.get(b, -1) for b in comp])
        if use_cfg_any:
            sched[0][:n_mix, comp, 0] = 1.0
            sched[0][:n_mix, comp, 1] = 0.0
        mix = ((list(range(B)) if use_cfg_any else []) + term_src + pag_src, [n_reg + j for j in range(len(term_src))], mix_rows,
               mix_coef)
    n_rows = (2 * B if use_cfg_any else B) + (len(mix[0]) - (B if use_cfg_any else 0) if mix is not None else 0)
    w_table = None
    if pag_src and torch.is_tensor(attn_weights):      # perturbed rows read their sample's row of a per-sample table
        attn_weights = [attn_weights] * B
    if isinstance(attn_weights, (list, tuple)):       # per-sample vectors, for the conditional rows only
        w_table = ops.attn_weights_table(attn_weights, B, [model.max_attn_weights((H, W), model.conditioning_seq_len(model_inputs))] * B)
    w_row = None
    if w_table is not None and pag_src:
        # one zero-length row (B) for the unconditional and term rows; perturbed row k reads row pag_src[k]
        w_table = (torch.cat([w_table[0], torch.zeros(1, w_table[0].shape[1])]), torch.cat([w_table[1], torch.zeros(1, dtype=torch.int32)]))
        w_row = torch.tensor(list(range(B)) + [B] * (n_rows - B - len(pag_src)) + pag_src, dtype=torch.int32)
    if ops.per_sample(generator):
        ops.check_generators(generator, B, dev)
        ops.check_per_sample_numel(H * W * model.num_labels)
    with torch.inference_mode():
        # one copy for the whole loop: [steps][B][3] params and [steps + 1][B] noise levels, a CPU region and the wrap table
        region_host = region is not None and region.device.type == "cpu"
        parts = (list(sched) if sched is not None else []) + (list(trunc) if trunc is not None else []) + ([region] if region_host else [])
        parts += [wrap] if wrap is not None else []
        parts += [torch.tensor(mix[0], dtype=torch.int32), mix[2], mix[3]] if mix is not None else []
        parts += [inj] if any(inj_steps) else []
        if pag_src:     # the per-row AttnBlock masks: zero before the perturbed rows, each perturbed row its sample's
            pag_rows = torch.zeros(n_rows, dtype=torch.int64)
            pag_rows[n_rows - len(pag_src):] = pag_t[1][pag_src]
            parts += [pag_rows] + ([w_row] if w_row is not None else [])
        parts += [conf] if conf is not None else []
        parts_d = ops.to_device_packed(parts, dev) if parts else []
        conf_d = parts_d.pop() if conf is not None else None
        w_row_d = parts_d.pop() if w_row is not None else None
        pag_rows_d = parts_d.pop() if pag_src else None
        inj_d = parts_d.pop() if any(inj_steps) else None
        if mix is not None:
            mix_coef_d, mix_rows_d, tail_d = parts_d.pop(), parts_d.pop(), parts_d.pop()
        wrap_d = parts_d.pop() if wrap is not None else None
        if sched is not None:
            params_d, r_d = parts_d[0], parts_d[1]
        trunc_d = (parts_d[2], parts_d[3]) if trunc is not None else None
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
        # an adapter is part of the model: a sample's unconditional, regional and term prompts are projected under its adapter
        glora = [entries] * len(groups) if lora_t is not None else None
        xlora = extra_lora if lora_t is not None else None
        # with guidance prompts the guided batch is [B conditional; B unconditional; term rows by sample, then term]
        cond_full = model.prepare_conditioning(groups, (H, W), extra=extra, tail=mix[1] if mix is not None else (), lora=glora,
                                               extra_lora=xlora, pag_tail=pag_src)
        if pag_src and not use_cfg_any:     # the steps without PAG: the conditional rows alone, on the same cache
            cond_plain = ConditioningCache(cond_full.cache, B, cond_full.s_max, cond_full.slots, cond_full.slot_map[:B],
                                           cond_full.extra_slot)
        regional_full = model.regional_device(regions, cond_full) if regions is not None else None
        extra_only = extra[:len(extra) - len(mix[1])] if mix is not None else extra
        lora_d = ops.lora_device(lora_t, dev)
        cond_only = regional_only = None
        # attention maps: the conditional rows [0, B) accumulate into rows [0, B), finalized once after the loop
        maps_len = model.conditioning_seq_len(model_inputs) if attention_maps else 0
        acc = model.map_accumulator(B, maps_len, (H, W)) if attention_maps else None
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
                    cond_only = model.prepare_conditioning([model_inputs], (H, W), extra=extra_only, lora=glora[:1] if glora else None,
                                                           extra_lora=xlora[:len(extra_only)] if xlora is not None else None)
                    regional_only = model.regional_device(regions, cond_only) if regions is not None else None
                cond, tokens = cond_only, sampled
            else:
                cond, tokens = (cond_full if not pag_src or i < n_mix else cond_plain), sampled
            if sched is None:
                r = torch.full((tokens.shape[0],), float(t_list[i]), dtype=torch.float32, device=dev)
                cfg_i, temp_i = (float(cfgs[i]) if guided else None), float(temperatures[i])
            else:
                r, params_i = r_d[i], params_d[i]
            composed = mix is not None and i < n_mix and (guided or not use_cfg_any)
            perturbed = composed and bool(pag_src)
            feats = model.features(tokens, r, cond, attn_weights, (n_rows if perturbed and w_row is not None else B)
                                   if attn_weights is not None else 0, cfg_pairs=guided and not composed, w_len=w_len,
                                   w_row=w_row_d if perturbed else None, wrap=wrap_d, regional=regional_only if cond is cond_only else regional_full,
                                   tail_src=tail_d if composed else None, maps=(None, B, acc) if attention_maps else None,
                                   inject=inj_d[i] if inj_steps[i] else None, lora=lora_d, perturb=pag_rows_d if perturbed else None)
            if composed:
                model.guidance_mix(feats, H * W, mix_rows_d, mix_coef_d[i])
            if step_modes is not None:
                sampled = _sample_modes_step(model, feats, B, H, W, guided, params_i, step_modes, generator, codebook, dev, trunc_d)
            elif mode == "multinomial" and not exact:
                if sched is None:
                    sampled = model.sample_tokens(feats, B, H, W, cfg_i, temp_i, generator)
                else:
                    sampled = model.sample_tokens_params(feats, B, H, W, guided, params_i, generator, trunc_d)
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
                if conf_d is not None:      # confidence from the operand the step's sampler read
                    logp = model.token_logprob(feats, B, B if guided else 0, H * W, params_i, sampled)
                    sampled = model.add_noise(sampled, t_next, random_x=init_noise, generator=generator, src=src_d if region_d is not None
                                              else None, region=region_d, confidence=logp, choice_temperature=conf_d)[0]
                elif region_d is None:
                    sampled = model.add_noise(sampled, t_next, random_x=init_noise, generator=generator)[0]
                else:
                    sampled = model.add_noise(sampled, t_next, random_x=init_noise, generator=generator, src=src_d, region=region_d)[0]
                if collect:
                    intermediates.append(sampled)
        maps = model.finalize_attention_maps(acc, (H, W), maps_len, steps) if attention_maps else None
    return sampled, intermediates, maps


def _sample_modes_step(model, feats, B, H, W, guided, params, step_modes, generators, codebook, dev, trunc=None):
    """One step of a batch whose samples are in different modes, on per-sample generators: the multinomial samples draw what
    a batch-1 step draws on their own generators, the others draw nothing.  The draws and the mode table go to the device in
    one asynchronous copy."""
    vals = []
    for g, md in zip(generators, step_modes):
        vals += ops.philox_values([g], H * W * model.num_labels, dev) if md == "multinomial" else [0, 0]
    seed_d, table_d = ops.to_device_packed([torch.tensor(vals, dtype=torch.int64).view(-1, 2), ops.mode_table(step_modes)], dev)
    return model.sample_tokens_modes(feats, B, B if guided else 0, H, W, params, seed_d, step_modes, table_d, codebook, trunc=trunc)


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


# utils.score: fp32 [B] mean nll, loss and argmax accuracy over the scored tokens, and the fp32 [B, H, W] per-token nll averaged
# over the levels
Scores = namedtuple("Scores", ["nll", "loss", "acc", "nll_map"])


def score(model, tokens, model_inputs, unconditional_inputs=None, levels=None, cfg=None, label_smoothing=0.0, generator=None,
          region=None, attn_weights=None, tiling=None, prompt_regions=None, lora=None) -> Scores:
    """The Monte-Carlo denoising score of ``tokens`` (int64 [B, H, W] on the model's device) under ``model_inputs``.

    For each noise level t_k of ``levels`` in order (default torch.linspace(1.0, 0.0, 9)[:8], the levels at which an 8-step
    sample() calls the model) the tokens are noised with exactly the draws of ``model.add_noise(tokens, t_k * ones(B),
    generator=generator)`` -- a mask, then the replacement codes, on the default CUDA generator, one generator, or per sample on
    a list of B -- and the noised grid is scored against ``tokens`` by ``model.token_scores`` at r = t_k, with ``cfg``,
    ``unconditional_inputs``, ``label_smoothing``, ``attn_weights``, ``tiling``, ``prompt_regions`` and ``lora`` as there.  ``region`` (bool
    [B, H, W] on the CPU or the model's device) keeps the tokens outside it from ever being noised (add_noise's ``src=tokens,
    region=region``) and restricts the means to the tokens inside it.

    Returns Scores(nll, loss, acc, nll_map): nll_map fp32 [B, H, W] is the levels' nll summed in level order in fp32 and divided by
    K = len(levels); nll and loss fp32 [B] are the means over the scored tokens of nll_map and of the levels' mean loss, and acc
    fp32 [B] is train.py's accuracy, the fraction of scored tokens and levels whose arg-max code is the token.  Rows with equal
    tokens, prompt and seed get equal scores where the forward is batch-invariant (DESIGN.md §3), so per-sample generators
    seeded alike compare prompts on common noise.  ValueError, before anything is enqueued and before any generator advances,
    for tokens that are not int64 [B, H, W] on the model's device, bad levels, an eps outside [0, 1], and a bad cfg,
    generator list, region, attn_weights, tiling, prompt_regions or lora."""
    dev = model._device()
    if not torch.is_tensor(tokens) or tokens.dim() != 3:
        raise ValueError("tokens: expected int64 codes [B, H, W] on the model's device")
    model._check_score_targets(tokens, tokens.shape, "tokens")
    B, H, W = tokens.shape
    levels = ops.check_score_levels(torch.linspace(1.0, 0.0, 9)[:8] if levels is None else levels)
    eps = ops.check_label_smoothing(label_smoothing)
    if ops.per_sample(generator):
        ops.check_generators(generator, B, dev)
        ops.check_per_sample_numel(H * W)
    check_region(region, tokens, tokens.shape, dev)
    setup = model._score_setup(B, (H, W), model_inputs, unconditional_inputs, cfg, attn_weights, tiling, prompt_regions, lora)
    region_d = region.to(dev) if region is not None else None
    nll_sum = loss_sum = hits = None
    for t_k in levels:
        t = torch.full((B,), t_k, dtype=torch.float32, device=dev)
        if region_d is None:
            noised = model.add_noise(tokens, t, generator=generator)[0]
        else:
            noised = model.add_noise(tokens, t, generator=generator, src=tokens, region=region_d)[0]
        s = model._score_tokens(setup, noised, t, tokens, eps)
        hit = (s.argmax == tokens).to(torch.float32)
        if nll_sum is None:
            nll_sum, loss_sum, hits = s.nll.clone(), s.loss.clone(), hit
        else:
            nll_sum += s.nll
            loss_sum += s.loss
            hits += hit
    K = len(levels)
    nll_map = nll_sum / K
    w = region_d.to(torch.float64) if region_d is not None else torch.ones(B, H, W, dtype=torch.float64, device=dev)
    n = w.sum((1, 2))

    def mean(m):
        return ((m.double() * w).sum((1, 2)) / n).float()
    return Scores(mean(nll_map), mean(loss_sum / K), mean(hits / K), nll_map)


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


def _decode_tail(tokens, decode, decode_output, tiling=None):
    """The step after the path (SURVEY.md §8 f2; ref/src_distributed/train.py:168-171, notebook nb:354-357): the final token
    grid goes straight into the f4 decoder on the same stream -- no host round trip, no separate clamp / byte pass."""
    if decode is None:
        return tokens
    if decode_output == "uint8":
        return decode.decode_indices_u8(tokens, tiling)
    if decode_output == "clamp":
        return decode.decode_indices_clamped(tokens, tiling)
    if decode_output == "raw":
        return decode.decode_indices(tokens, tiling)
    raise ValueError(f"decode_output={decode_output!r}: expected 'uint8', 'clamp' or 'raw'")


def sample(model, model_inputs, latent_shape, unconditional_inputs=None, steps=12, renoise_steps=11, temperature=(1.0, 0.2),
           cfg=8.0, t_start=1.0, t_end=0.0, device="cuda", exact=False, decode=None, decode_output="uint8", generator=None,
           top_k=None, top_p=None, tiling=None, prompt_regions=None, guidance_prompts=None, attention_maps=False,
           attention_source=None, lora=None, pag=None, confidence_renoise=None):
    """ref/src/utils.py:35-55 (same positional/keyword arguments; ``device`` is accepted and must be the model's).
    ``exact=True`` materialises the logits and uses the op-for-op torch arithmetic (parity path).
    ``decode=vqmodel`` appends the reference callers' next step, ``vqmodel.decode_indices(tokens).clamp(0, 1)``, fused on the
    tail: returns uint8 NHWC images (``decode_output='uint8'``), clamped fp32 NCHW ('clamp') or unclamped fp32 NCHW ('raw').
    ``generator``: None draws on the default CUDA generator; one CUDA ``torch.Generator`` replaces it; a list of B of them gives
    every sample its own stream -- row i draws what this call with batch 1 on sample i's inputs draws after
    ``torch.manual_seed(generator[i].initial_seed())`` (and equals it where the forward is batch-invariant, DESIGN.md §3),
    and leaves generator i where that call leaves the default generator.
    Per-sample settings (module docstring): ``cfg`` [B], ``temperature`` [B, 2], ``t_start`` / ``t_end`` [B].  A per-sample cfg
    of 0 is unguided like the scalar ``cfg=0``; so is 1.0, and an all-zero tensor makes the whole call unguided.
    ``top_k`` / ``top_p`` (module docstring): None, a scalar, or a CPU tensor [B]; ValueError, before anything is enqueued and
    before any generator advances, for a bad value and for truncation with exact=True.
    ``tiling`` (module docstring): seamless tiling per call or per sample; with ``decode`` each image is decoded with its own
    tiling.  ValueError, before anything is enqueued and before any generator advances, for an unknown value, a list of the
    wrong length or a tensor.  ``prompt_regions`` (module docstring): regional prompts per sample.  ``guidance_prompts`` (module
    docstring): weighted extra and negative prompts per sample in the guided mix; a sample with terms needs a cfg other than 0.
    ``attention_maps=True`` (module docstring): returns (tokens or images, maps).  ``attention_source`` (module docstring):
    prompt-to-prompt edits of other samples of the call; give each edit its own generator seeded like its source's.
    ``lora`` (module docstring): a LoRA adapter per sample, or one for every sample.  ``pag`` (module docstring):
    perturbed-attention guidance per sample, with CFG or without it.  ``confidence_renoise`` (module docstring): renoise each
    sample's least likely tokens, one choice temperature for every sample or one entry per sample."""
    ops.check_attention_maps(attention_maps, prompt_regions)
    per_sample_cfg = torch.is_tensor(cfg)
    terms = ops.guidance_table(guidance_prompts, latent_shape[0])
    if terms is not None and per_sample_cfg:
        for b, v in enumerate(ops.per_sample_values("cfg", cfg, latent_shape[0])):
            if terms[b] and not v:
                raise ValueError(f"guidance_prompts[{b}]: a sample with guidance prompts needs a cfg other than 0 (unguided)")
    if per_sample_cfg:
        cfg_vals = [v if v else 1.0 for v in ops.per_sample_values("cfg", cfg, latent_shape[0])]   # f*1 + u*0 = f
        cfgs = [[v] * steps for v in cfg_vals] if any(cfg.tolist()) else None
        per_sample_cfg = cfgs is not None
    else:
        cfgs = [cfg] * steps if cfg else None
    if cfgs is not None and unconditional_inputs is None:
        raise TypeError("sample(): cfg is set but unconditional_inputs is None")
    out, _, maps = _sample_core(model, model_inputs, tuple(latent_shape), unconditional_inputs, None, steps, renoise_steps,
                                temperature, cfgs, t_start, t_end, steps, "multinomial", None, exact, False, generator=generator,
                                per_sample_cfg=per_sample_cfg, top_k=top_k, top_p=top_p, tiling=tiling,
                                prompt_regions=prompt_regions, guidance_prompts=guidance_prompts, attention_maps=attention_maps,
                                attention_source=attention_source, lora=lora, pag=pag, confidence_renoise=confidence_renoise)
    out = _decode_tail(out, decode, decode_output, tiling)
    return (out, maps) if attention_maps else out


def sample_distributed(model, model_inputs, unconditional_inputs, latent_shape, init_x=None, steps=12, renoise_steps=None,
                       temperature=(0.7, 0.3), cfg=(8.0, 8.0), t_start=1.0, t_end=0.0, sampling_conditional_steps=None,
                       exact=False, generator=None, region=None, top_k=None, top_p=None, tiling=None, prompt_regions=None,
                       guidance_prompts=None, attention_maps=False, attention_source=None, lora=None, pag=None,
                       confidence_renoise=None):
    """ref/src_distributed/utils.py:97-126.  ``generator`` as in ``sample``: a shard given ``generators[lo:hi]`` draws what
    rows [lo, hi) of the single-GPU call draw.  Per-sample settings (module docstring): ``cfg`` and ``temperature`` [B, 2],
    ``t_start`` / ``t_end`` [B]; a shard given ``settings[lo:hi]`` computes what rows [lo, hi) compute.  ``region`` (module
    docstring): bool [B, H, W] on the CPU or the model's device, True where tokens are generated; ``init_x`` then holds the
    tokens kept elsewhere.  ValueError, before anything is enqueued and before any generator advances, for a region without
    init_x, of another shape or dtype, or on another device.  ``top_k`` / ``top_p`` as in ``sample``; a shard given
    ``top_k[lo:hi]`` computes what rows [lo, hi) compute.  ``tiling`` as in ``sample``; a shard given ``tiling[lo:hi]`` computes
    what rows [lo, hi) compute.  ``prompt_regions`` (module docstring) likewise: a shard given ``prompt_regions[lo:hi]`` computes
    what rows [lo, hi) compute.  ``guidance_prompts`` (module docstring) likewise: a shard given ``guidance_prompts[lo:hi]``
    computes what rows [lo, hi) compute.  ``attention_maps=True`` (module docstring): returns (tokens, maps) for the shard's rows.
    ``attention_source`` (module docstring): a source and its edits sit in the same shard, with indices relative to the shard.
    ``lora`` (module docstring): a shard given ``lora[lo:hi]`` computes what rows [lo, hi) compute; each rank loads its adapters
    itself (load_lora).  ``pag`` (module docstring) likewise: a shard given ``pag[lo:hi]`` computes what rows [lo, hi) compute.
    ``confidence_renoise`` (module docstring) likewise: a shard given ``confidence_renoise[lo:hi]`` computes what rows [lo, hi)
    compute."""
    ops.check_attention_maps(attention_maps, prompt_regions)
    if sampling_conditional_steps is None:
        sampling_conditional_steps = steps
    if renoise_steps is None:
        renoise_steps = steps - 1
    cfgs = _cfg_schedule(cfg, latent_shape[0], steps)
    out, _, maps = _sample_core(model, model_inputs, tuple(latent_shape), unconditional_inputs, init_x, steps, renoise_steps,
                                temperature, cfgs, t_start, t_end, sampling_conditional_steps, "multinomial", None, exact, False,
                                generator=generator, per_sample_cfg=torch.is_tensor(cfg), region=region, top_k=top_k, top_p=top_p,
                                tiling=tiling, prompt_regions=prompt_regions, guidance_prompts=guidance_prompts,
                                attention_maps=attention_maps, attention_source=attention_source, lora=lora, pag=pag,
                                confidence_renoise=confidence_renoise)
    return (out, maps) if attention_maps else out


def sample_notebook(model, model_inputs, latent_shape, unconditional_inputs=None, init_x=None, steps=12, renoise_steps=None,
                    temperature=(0.7, 0.3), cfg=(8.0, 8.0), mode='multinomial', t_start=1.0, t_end=0.0,
                    sampling_conditional_steps=None, sampling_quant_steps=None, attn_weights=None, exact=False, vqmodel=None,
                    generator=None, region=None, top_k=None, top_p=None, tiling=None, prompt_regions=None, guidance_prompts=None,
                    attention_maps=False, attention_source=None, lora=None, pag=None, confidence_renoise=None):
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
    nothing, the multinomial ones draw per sample); one whose entries are all equal is the scalar call (sampling_modes).
    ``top_k`` / ``top_p`` as in ``sample``: they truncate the multinomial steps only.  ``tiling`` as in ``sample``: the
    intermediates are those of the tiled call.  ``prompt_regions`` as in ``sample``; regional samples' rows may not also
    have ``attn_weights``.  ``guidance_prompts`` as in ``sample``: the argmax and quant steps of a sample with terms see its mixed
    features, and ``attn_weights`` weight its conditional row only.  ``attention_maps=True`` (module docstring): returns
    (sampled, intermediate_images, maps).  ``attention_source`` (module docstring): prompt-to-prompt edits; an edit's
    ``attn_weights`` reweight the replayed probabilities.  ``lora`` (module docstring): a LoRA adapter per sample.  ``pag``
    (module docstring): perturbed-attention guidance per sample; its perturbed row carries the sample's ``attn_weights``, and the
    argmax and quant steps see the mixed features.  ``confidence_renoise`` (module docstring): renoise each sample's least likely
    tokens; the intermediates show the renoised grids."""
    ops.check_attention_maps(attention_maps, prompt_regions)
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
    sampled, intermediates, maps = _sample_core(model, model_inputs, tuple(latent_shape), unconditional_inputs, init_x, steps,
                                                renoise_steps, temperature, cfgs, t_start, t_end, sampling_conditional_steps, mode,
                                                attn_weights, exact, True, sampling_quant_steps, codebook, generator,
                                                per_sample_cfg=torch.is_tensor(cfg), region=region, modes=modes, top_k=top_k,
                                                top_p=top_p, tiling=tiling, prompt_regions=prompt_regions,
                                                guidance_prompts=guidance_prompts, attention_maps=attention_maps,
                                                attention_source=attention_source, lora=lora, pag=pag,
                                                confidence_renoise=confidence_renoise)
    return (sampled, intermediates, maps) if attention_maps else (sampled, intermediates)
