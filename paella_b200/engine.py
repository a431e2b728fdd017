"""SamplingEngine: step-level batching of ``sample_distributed`` requests.

A ``sample()`` call is a closed batch: its requests start together, share one step count, and the call returns when the
longest schedule is done.  The engine instead admits and retires requests at every step, so requests with different step
counts, settings and arrival times share one denoiser batch:

    eng = SamplingEngine(model, latent_hw=(32, 32), max_batch=64, max_cond_len=140)
    req = eng.submit(inputs, uncond, generator=g, steps=12, cfg=(8.0, 8.0))
    while eng.busy:
        for r in eng.step():        # the requests that finished in this step
            use(r.result)           # a device tensor, ordered on the current stream

A request's tokens are those of ``sample_distributed(model, inputs, uncond, (1, H, W), init_x, steps, renoise_steps,
temperature, cfg, t_start, t_end, sampling_conditional_steps, generator=[g])``: the same draws from ``g`` in the same order
(randint at admission, then per step the sampler's exponential draw and, if the step renoises, the mask draw), the same
torch.linspace schedules and fp32 kernel constants (utils.sampling_schedule), and ``g`` left at the same offset.  Where the
forward is batch-invariant (DESIGN.md §3: on the default model with ``model.batch_invariant = True``) the tokens are equal
bit for bit, whatever else is in flight.  With
``attn_weights=w`` (and ``keep_intermediates=True``) the request's tokens, ``req.intermediates`` and generator offset are those
of ``sample_notebook(model, inputs, (1, H, W), uncond, init_x, steps, renoise_steps, temperature, cfg, 'multinomial', t_start,
t_end, sampling_conditional_steps, attn_weights=w, generator=[g])``; each step's batch reads every row's weights from a
device pool indexed by its token slot.  With ``region=`` (bool [1, H, W], True where tokens are generated) and ``init_x`` (the
source tokens kept elsewhere) a request inpaints or outpaints as ``sample_distributed(..., init_x, region=region)`` does: its
source tokens and region sit in device pools by token slot, and the step's one add-noise launch puts every row's source
tokens back outside its region (a request without a region has an all-True row).  With ``mode='argmax'`` or ``'quant'`` and
``sampling_quant_steps=k`` (steps i >= k use 'quant'; 'quant' needs the engine's ``vqmodel``) the request's tokens, intermediates
and generator offset are those of ``sample_notebook(model, inputs, (1, H, W), uncond, init_x, steps, renoise_steps, temperature,
cfg, mode, t_start, t_end, sampling_conditional_steps, sampling_quant_steps, attn_weights, vqmodel=vq, generator=[g],
region=region)``: a step in argmax or quant mode draws nothing from ``g`` (only its mask draw, if it renoises).  With
``top_k`` / ``top_p`` a request's multinomial steps are truncated as in ``sample_notebook(..., top_k=k, top_p=p)``; the draws,
and so the generator offsets, are those of the untruncated request.  With ``tiling='x'``, ``'y'`` or ``'xy'`` a request's token
grid wraps around as in ``sample_notebook(..., tiling=t)`` (seamless textures and panoramas), and ``decode=True`` decodes it
with the same tiling; tiling draws nothing.  With ``prompt_regions=[(inputs, region), ...]`` (an engine built with
``max_prompt_regions`` > 0) a request carries regional prompts as ``sample_notebook(..., prompt_regions=[regions])`` does: their
K/V are projected at admission into slots reserved for its token slot, and its token masks and region slots sit in device
pools by token slot; regional prompts draw nothing.  With ``guidance_prompts=[(inputs, weight), ...]`` (an engine built with
``max_guidance_prompts`` > 0) a guided request mixes further weighted prompts into its guidance as ``sample_notebook(...,
guidance_prompts=[terms])`` does: their K/V are projected at admission into slots reserved for its token slot, and each of its
guided steps runs one more denoiser row per term; terms draw nothing.  With ``attention_maps=True`` a request's
``req.attention_maps`` (float32 [S, H, W], S its conditioning length) is set when it retires, equal bit for bit to the maps of
``sample_notebook(..., attention_maps=True)`` on the same request; its tokens are unchanged, and maps draw nothing.  With
``attention_source=(src, k)`` a request is a prompt-to-prompt edit of the queued request ``src``: the edit and its source are
admitted together and advance in lockstep, and on its steps i < k the edit's conditional forward replays the source's attention
probabilities, as ``sample_notebook(..., attention_source=[None, (0, k)])`` does on the pair; injection draws nothing.  With
``lora=adapter`` or ``(adapter, scale)`` a request runs under a LoRA adapter as ``sample_notebook(..., lora=[entry])`` does: its
K/V slots are projected under the adapter at admission, and a guided request without a negative prompt of its own gets its own
unconditional slot, holding the engine-wide unconditional inputs projected under its adapter (the shared slot is the model's
without an adapter); adapters draw nothing.  One step's launches take at most 32 distinct adapters (ops.MAX_LORA_ADAPTERS):
admission holds a request whose adapter would be the 33rd in flight, and everything queued behind it, until a request retires.
With ``pag=s`` or ``(s, blocks)`` a request gets perturbed-attention guidance as ``sample_notebook(..., pag=[entry])`` does: on each
of its steps before sampling_conditional_steps, guided or not, one more denoiser row -- its perturbed forward, reading its own
conditional slot, weight row, wrap byte and adapter -- follows the term rows, and its mix coefficients (c + s, ..., -s) ride in
the step table with the row's AttnBlock mask; PAG draws nothing and needs no K/V slot.  With ``confidence_renoise=tau`` a request
renoises its least likely tokens as ``sample_notebook(..., confidence_renoise=[tau])`` does (utils module docstring): on the
request's renoising steps its tokens' log-probabilities come from the step's sampler operand (Paella.token_logprob) and its
mask from the uniforms of its own mask draw; it draws nothing more.

Each step orders its batch with the guided requests first: rows [0, n_pairs) are guided, [n_pairs, Bc) are not, and the
unconditional rows of the guided ones follow as [Bc, Bc + n_pairs) (Paella.features with ``n_pairs``).  Per step the host
builds one table (noise levels, (cfg, 1 - cfg, 1/T), renoise targets, Philox (seed, offset) pairs, row -> slot maps) and
sends it to the device with one asynchronous copy; the step itself is a gather of the rows from the token pool, the forward,
one fused-sampler launch and one per-sample add-noise launch that writes every row back into its slot.  A step whose rows are
in several sampling modes adds each row's mode to the table: the fused sampler skips the argmax and quant rows, which then go
through the out_mapper GEMM to logits (a bounded number of samples at a time) and the argmax or quant kernel, one call per mode
(Paella.sample_tokens_modes).  A step in which some request truncates adds each row's (k, p) to the table, and the fused sampler
reads them there (0 and 1.0 for the rows that do not); a step in which none does launches exactly as without truncation.  A step
in which some row tiles adds each row's wrap byte (0 for the rows that do not), read by the denoiser's depthwise convolutions; a
step in which none does launches exactly as without tiling.  A step in which some row is regional launches the regional
denoiser (pb200_paella_features_regional), each row reading its token slot's masks and region slots; a step in which none is
launches exactly as without regional prompts.  A step in which some guided row has guidance prompts appends their term rows after
the unconditional rows, ordered by request, then term (pb200_paella_features_tail, each term row reading its own K/V slot), mixes
each such request's rows into its conditional row (pb200_paella_guidance_mix) and samples that row with the params (1, 0, 1/T); the
tail map, mix rows and coefficients ride in the step's table.  A step with no such row launches exactly as without them.  A
step in which some row wants attention maps adds each row's map row (its token slot, -1 for the rows that do not) to the table and
runs the maps denoiser (pb200_paella_features_maps), which accumulates into a pool of per-slot accumulators, allocated when the
first such request is admitted and zeroed per request at admission; a request's maps are finalized with its own step count when it
retires.  A step with no such row launches exactly as without maps.  A step in which some edit is inside its window adds each
row's source row in this step's order (-1 for the other rows) to the table and runs the injecting denoiser
(pb200_paella_features_inject); a step with no such row launches exactly as without edits.  A step in which some row has a LoRA
adapter adds each row's adapter index and scale to the table and runs the adapted denoiser (pb200_paella_features_lora); a step
with no such row launches exactly as without adapters.  No adapter memory is reserved: an adapter lives in its LoraAdapter.  A
step in which some renoising row has a choice temperature adds each row's (-1 for the others) to the table, scores the step's drawn
tokens (pb200_paella_token_logprob) and renoises every row in one pb200_renoise_confidence_per_sample launch in place of the
add-noise launch, the other rows by add_noise's rule; a step with no such row launches exactly as without it.
The host knows which
requests finish at which step, so ``step()`` never synchronises.  Admission projects the conditioning of the requests admitted
in one step together: one prepare_cond per run of contiguous slots with one sequence layout (``admission_runs``), conditional
and own unconditional slots alike; the cache rows equal per-request projections bit for bit in either mode.
"""
from __future__ import annotations

import collections
from typing import Dict, List, Optional, Tuple

import torch

from . import ops
from . import utils as U
from ._lib import lib
from .modules import ConditioningCache, Paella


class Request:
    """One submitted request.  ``result`` is set (a device tensor) in the ``step()`` that retires it: int64 tokens [1, H, W],
    or with ``decode=True`` the uint8 NHWC image [1, 4H, 4W, 3].  With ``keep_intermediates=True``, ``intermediates`` grows by
    the sampled tokens of every step, then the renoised tokens if the step renoises."""

    def __init__(self, steps: int, renoise_steps: int, cond_steps: int, guided: bool, params: torch.Tensor, r: torch.Tensor,
                 generator=None, inputs=None, uncond=None, init_x=None, decode: bool = False,
                 attn_weights: Optional[torch.Tensor] = None, keep_intermediates: bool = False,
                 region: Optional[torch.Tensor] = None, mode: str = "multinomial", quant_steps: Optional[int] = None,
                 top_k: int = 0, top_p: float = 1.0, wrap: int = 0, regions=None, terms=None, mix_coef=None,
                 attention_maps: bool = False, maps_len: int = 0, attention_source=None, lora=None, pag=None, confidence: float = -1.0):
        self.steps, self.renoise_steps, self.cond_steps, self.guided = steps, renoise_steps, cond_steps, guided
        self.params, self.r = params, r          # CPU float32 [steps, 3] and [steps + 1]: rows of utils.sampling_schedule
        self.generator, self.inputs, self.uncond, self.init_x, self.decode = generator, inputs, uncond, init_x, decode
        self.attn_weights = attn_weights         # CPU float32 [n] or None
        self.region = region                     # bool [1, H, W] or None, until admission
        self.has_region = region is not None
        self.mode, self.quant_steps = mode, quant_steps      # sampling mode, and the step from which 'quant' is used (or None)
        self.top_k, self.top_p = top_k, top_p    # the truncation table's row: 0 and 1.0 are off
        self.wrap = wrap                         # the wrap table's byte (ops.tiling_table): bit 0 x, bit 1 y; 0 is off
        self.regions = regions                   # regional prompts: (uint8 [H, W] token masks, [inputs, ...]) or None
        self.regional = regions is not None
        self.terms = terms                       # guidance prompts: [(inputs, weight), ...] until admission, or None
        self.n_terms = len(terms) if terms is not None else 0
        self.mix_coef = mix_coef                 # CPU float32 [cond_steps, row width]: the mixed steps' coefficients (guided:
        #                                          c, u, the terms, then -s with PAG; unguided with PAG: 1 + s, -s)
        self.pag = pag                           # perturbed-attention guidance: (scale, int64 AttnBlock mask) or None
        self.confidence = confidence             # confidence-guided renoising: the choice temperature, -1 for none
        self.term_slot: List[int] = []           # the K/V slots of the terms
        self.want_maps, self.maps_len = attention_maps, maps_len      # attention maps, over maps_len conditioning keys
        self.attention_maps: Optional[torch.Tensor] = None            # float32 [maps_len, H, W], set at retirement
        # prompt-to-prompt: the source request and the steps it is replayed on, or None; a source lists its edits
        self.inj_src, self.inj_k = attention_source if attention_source is not None else (None, 0)
        self.edits: List["Request"] = []
        self.lora = lora                         # LoRA: (adapter, scale) or None, held until retirement
        # with keep_intermediates: what sample_notebook returns as its second value, device tensors [1, H, W]
        self.intermediates: Optional[List[torch.Tensor]] = [] if keep_intermediates else None
        self.k = 0                               # steps done
        self.slot: Optional[int] = None          # token pool slot and conditional K/V slot
        self.uncond_slot: Optional[int] = None   # unconditional K/V slot
        self.result: Optional[torch.Tensor] = None

    @property
    def done(self) -> bool:
        return self.result is not None

    def mode_at(self, k: int) -> str:
        """The sampling mode of step k: 'quant' from step ``sampling_quant_steps`` on, the request's own mode before."""
        return ops.mode_at(self.mode, self.quant_steps, k)


class StepPlan:
    """The host tables of one step (CPU tensors), rows in batch order: guided requests first.  ``w_zero_row``: the weight-pool
    row of length 0 that the unconditional and term rows of a perturbing step read."""

    def __init__(self, order: List[Request], w_zero_row: int = -1):
        self.order = order
        self.n_pairs = sum(1 for q in order if q.guided and q.k < q.cond_steps)
        Bc, n_pairs = len(order), self.n_pairs
        # perturbed-attention guidance: the rows perturbed this step (guided or not, before their sampling_conditional_steps)
        self.perturbed = [i for i, q in enumerate(order) if q.pag is not None and q.k < q.cond_steps]
        pert = set(self.perturbed)
        # guidance prompts and PAG: the composed rows -- guided rows with terms or PAG, unguided rows with PAG -- then their term
        # rows after the unconditional rows, then their perturbed rows
        self.composed = [i for i, q in enumerate(order) if (i < n_pairs and q.n_terms) or i in pert]
        term_src = [i for i in self.composed if i < n_pairs for _ in range(order[i].n_terms)]
        self.tail = torch.tensor(list(range(n_pairs)) + term_src + self.perturbed, dtype=torch.int32)
        p_row = {i: Bc + n_pairs + len(term_src) + j for j, i in enumerate(self.perturbed)}
        own = []
        t = Bc + n_pairs
        for i in self.composed:
            q = order[i]
            if i < n_pairs:
                own.append([i, Bc + i] + list(range(t, t + q.n_terms)) + ([p_row[i]] if i in pert else []))
                t += q.n_terms
            else:
                own.append([i, p_row[i]])
        width = max((len(o) for o in own), default=2)
        self.mix_rows = torch.full((len(self.composed), width), -1, dtype=torch.int32)
        self.mix_coef = torch.zeros(len(self.composed), width, dtype=torch.float32)
        for y, (i, o) in enumerate(zip(self.composed, own)):
            self.mix_rows[y, :len(o)] = torch.tensor(o, dtype=torch.int32)
            self.mix_coef[y, :len(o)] = order[i].mix_coef[order[i].k]
        n_rows = Bc + self.tail.numel()
        self.pag_rows = torch.zeros(n_rows, dtype=torch.int64)     # each row's AttnBlock mask, 0 but on the perturbed rows
        for i in self.perturbed:
            self.pag_rows[p_row[i]] = order[i].pag[1]
        # a perturbed row reads its request's weight row; the unconditional and term rows read the empty one
        self.pag_w_row = torch.tensor([q.slot if q.slot is not None else -1 for q in order] +
                                      [w_zero_row] * (n_rows - Bc - len(self.perturbed)) +
                                      [order[i].slot if order[i].slot is not None else -1 for i in self.perturbed], dtype=torch.int32)
        self.r = torch.stack([q.r[q.k] for q in order])
        self.params = torch.stack([q.params[q.k] for q in order])
        self.renoise = [q.k < q.renoise_steps for q in order]
        self.modes = [q.mode_at(q.k) for q in order]
        self.draws = [md == "multinomial" for md in self.modes]     # only multinomial rows draw the sampler's exponentials
        # the truncation table, when a row that draws truncates (otherwise the step launches without one)
        self.truncates = any(dr and (q.top_k > 0 or q.top_p < 1.0) for q, dr in zip(order, self.draws))
        self.top_k = torch.tensor([q.top_k for q in order], dtype=torch.int32)
        self.top_p = torch.tensor([q.top_p for q in order], dtype=torch.float32)
        # the wrap table, when some row tiles (otherwise the step launches the untiled kernels)
        self.wraps = any(q.wrap for q in order)
        self.wrap = torch.tensor([q.wrap for q in order], dtype=torch.uint8)
        # a row that does not renoise keeps its tokens (t < 0 never passes the mask test)
        self.t_next = torch.stack([q.r[q.k + 1] if rn else torch.tensor(-1.0) for q, rn in zip(order, self.renoise)])
        self.row_slot = torch.tensor([q.slot for q in order], dtype=torch.int32)
        self.kv_slot = torch.tensor([q.slot for q in order] + [q.uncond_slot for q in order[:self.n_pairs]] +
                                    [s for i in self.composed if i < n_pairs for s in order[i].term_slot] +
                                    [order[i].slot for i in self.perturbed], dtype=torch.int32)
        # attention maps: each row's accumulator row (its token slot), -1 for the rows without maps
        self.maps = any(q.want_maps for q in order)
        self.map_row = torch.tensor([q.slot if q.want_maps else -1 for q in order], dtype=torch.int32)
        # prompt-to-prompt: each edit inside its window reads its source's row of this step's order, -1 for the other rows
        row = {id(q): i for i, q in enumerate(order)}
        self.inj_src = torch.tensor([row[id(q.inj_src)] if q.inj_src is not None and q.k < q.inj_k else -1 for q in order],
                                    dtype=torch.int32)
        self.injects = bool((self.inj_src >= 0).any())
        # LoRA: each row's index into the step's distinct adapters (-1: none) and its scale, when some row has an adapter
        self.adapters, self.lora_id, self.lora_scale = ops.lora_rows([q.lora for q in order])
        self.loras = bool(self.adapters)
        # confidence-guided renoising: each row's choice temperature (-1: add_noise's rule), when some renoising row has one
        self.confident = any(rn and q.confidence >= 0 for q, rn in zip(order, self.renoise))
        self.tau = torch.tensor([q.confidence for q in order], dtype=torch.float32)


def cond_layout(inputs: Dict[str, torch.Tensor]) -> Tuple[int, bool, int]:
    """The sequence layout of one request's conditioning: (byt5 length, clip present, number of clip images).  Requests with
    one layout have the same sequence length and the same mapper launches, so they can be projected as one batch."""
    ci = inputs.get("clip_image")
    n_img = 0 if ci is None else (len(ci) if isinstance(ci, (list, tuple)) else 1)
    return int(inputs["byt5"].shape[1]), inputs.get("clip") is not None, n_img


def admission_runs(writes: List[Tuple[int, Tuple[int, bool, int]]]) -> List[List[int]]:
    """Group the conditioning writes of one admission -- (cache slot, layout) pairs with distinct slots -- into runs of
    contiguous slots that share one layout, in ascending slot order.  Each run is a list of indices into ``writes`` and is
    projected by one prepare_cond call at its first slot."""
    runs: List[List[int]] = []
    for i in sorted(range(len(writes)), key=lambda i: writes[i][0]):
        if runs and writes[i][0] == writes[runs[-1][-1]][0] + 1 and writes[i][1] == writes[runs[-1][-1]][1]:
            runs[-1].append(i)
        else:
            runs.append([i])
    return runs


def step_host_table(plan: StepPlan, draw: List[int], renoise: List[int]) -> Tuple[torch.Tensor, Dict[str, Tuple[str, int, int]]]:
    """The step's one host-to-device buffer: int64 [(seed, offset) pairs of the sampler's draw, then of the mask draw], then the
    float32 part [r, params (3 per row), t_next, (top_p), (mix_coef), (lora_scale), (tau)], then the int32 part [row_slot, kv_slot, (mode
    table), (top_k), (tail, mix_rows), (map_row), (inj_src), (lora_id), (w_row)], then the uint8 part [(wrap)], each part padded to
    whole int64 words, then (pag): the int64 AttnBlock mask of every row, tail included, with w_row (each row's weight-pool row)
    only when some row is perturbed this step (perturbed-attention guidance).  top_p / top_k are present only when ``plan.truncates``, the mode table only when the step mixes modes, wrap (one
    byte per row) only when ``plan.wraps``, the tail map and the mix table only when some row of the step is composed (guidance
    prompts), map_row only when some row wants attention maps, inj_src only when some edit is inside its window, lora_id and
    lora_scale only when some row has a LoRA adapter (the adapters' blob pointers travel as kernel arguments), tau only when some
    renoising row has a choice temperature (confidence-guided renoising).  Returns (buffer, {name: (dtype, start, length)}), start and length in elements of that dtype within its part."""
    Bc, n_pairs = len(plan.order), plan.n_pairs
    mixed = not all(plan.draws)
    modes = ops.mode_table(plan.modes) if mixed else torch.zeros(0, dtype=torch.int32)
    f32_parts = [("r", plan.r), ("params", plan.params.view(-1)), ("t_next", plan.t_next)]
    i32_parts = [("row_slot", plan.row_slot), ("kv_slot", plan.kv_slot), ("modes", modes)]
    if plan.truncates:
        f32_parts.append(("top_p", plan.top_p))
        i32_parts.append(("top_k", plan.top_k))
    if plan.composed:
        f32_parts.append(("mix_coef", plan.mix_coef.view(-1)))
        i32_parts += [("tail", plan.tail), ("mix_rows", plan.mix_rows.view(-1))]
    if plan.maps:
        i32_parts.append(("map_row", plan.map_row))
    if plan.injects:
        i32_parts.append(("inj_src", plan.inj_src))
    if plan.loras:
        f32_parts.append(("lora_scale", plan.lora_scale))
        i32_parts.append(("lora_id", plan.lora_id))
    if plan.perturbed:
        i32_parts.append(("w_row", plan.pag_w_row))
    if plan.confident:
        f32_parts.append(("tau", plan.tau))
    u8_parts = [("wrap", plan.wrap)] if plan.wraps else []
    layout: Dict[str, Tuple[str, int, int]] = {}
    for dt, parts in (("f32", f32_parts), ("i32", i32_parts), ("u8", u8_parts)):
        o = 0
        for name, v in parts:
            layout[name] = (dt, o, v.numel())
            o += v.numel()
    f32 = torch.cat([v for _, v in f32_parts])
    i32 = torch.cat([v for _, v in i32_parts])
    f32 = torch.cat([f32, torch.zeros(f32.numel() % 2)])
    i32 = torch.cat([i32, torch.zeros(i32.numel() % 2, dtype=torch.int32)])
    u8 = torch.cat([v for _, v in u8_parts] + [torch.zeros(0, dtype=torch.uint8)])
    u8 = torch.cat([u8, torch.zeros(-u8.numel() % 8, dtype=torch.uint8)])
    pag = plan.pag_rows if plan.perturbed else torch.zeros(0, dtype=torch.int64)
    host = torch.cat([torch.tensor(draw + renoise, dtype=torch.int64), f32.view(torch.int64), i32.view(torch.int64),
                      u8.view(torch.int64), pag])
    layout["f32"] = ("i64", 4 * Bc, f32.numel() // 2)
    layout["i32"] = ("i64", 4 * Bc + f32.numel() // 2, i32.numel() // 2)
    layout["u8"] = ("i64", 4 * Bc + f32.numel() // 2 + i32.numel() // 2, u8.numel() // 8)
    if plan.perturbed:
        layout["pag"] = ("i64", 4 * Bc + f32.numel() // 2 + i32.numel() // 2 + u8.numel() // 8, pag.numel())
    return host, layout


def _cat_inputs(inputs: List[Dict[str, torch.Tensor]], dev) -> Dict[str, torch.Tensor]:
    """Batch-1 conditioning dicts of one layout -> one batch, on ``dev``."""
    if len(inputs) == 1:
        return inputs[0]

    def cat(ts):
        return torch.cat([t.to(device=dev, dtype=torch.float32, non_blocking=True) for t in ts])
    out = {"byt5": cat([x["byt5"] for x in inputs])}
    if inputs[0].get("clip") is not None:
        out["clip"] = cat([x["clip"] for x in inputs])
    if inputs[0].get("clip_image") is not None:
        per = [list(ci) if isinstance(ci, (list, tuple)) else [ci] for ci in (x["clip_image"] for x in inputs)]
        out["clip_image"] = [cat([p[j] for p in per]) for j in range(len(per[0]))]
    return out


def admit_from_queue(queue: "collections.deque[Request]", n_free: int, active: List[Request] = ()) -> List[Request]:
    """Take the requests one admission starts from ``queue``, FIFO, into at most ``n_free`` slots.  A source comes in with
    every edit queued for it (its edits are queued after it), or it and everything behind it waits until enough slots are
    free.  Likewise a request whose LoRA adapter would take the adapters in flight (``active``'s and the admitted ones') past
    ops.MAX_LORA_ADAPTERS, the most one step's launches take, waits with everything behind it until a request retires."""
    new: List[Request] = []
    adapters = ops.distinct_adapters([q.lora for q in active])
    while queue and n_free - len(new) >= 1 + len(queue[0].edits):
        group = [queue[0]] + queue[0].edits
        grown = adapters + [a for a in ops.distinct_adapters([q.lora for q in group]) if not any(a is b for b in adapters)]
        if len(grown) > ops.MAX_LORA_ADAPTERS:
            break
        adapters = grown
        for q in group:
            queue.remove(q)
        new += group
    return new


def build_step_plan(active: List[Request], w_zero_row: int = -1) -> StepPlan:
    """Order the active requests for one step -- guided this step first, each group in admission order -- and build the
    step's tables from each request's own schedule rows at its own step index."""
    guided = [q for q in active if q.guided and q.k < q.cond_steps]
    return StepPlan(guided + [q for q in active if not (q.guided and q.k < q.cond_steps)], w_zero_row)


class SamplingEngine:
    """Step-level batcher over one Paella model and one latent grid (module docstring).

    ``max_batch`` requests are in flight at most; later ones queue and are admitted FIFO at step boundaries.  Conditioning of
    up to ``max_cond_len`` rows.  ``unconditional_inputs`` (batch 1) is projected once and used by every guided request that
    brings no negative prompt of its own.  ``vqmodel`` decodes the requests submitted with ``decode=True``.
    ``max_prompt_regions`` (0 .. 7): the regional prompts a request may carry.  The engine reserves that many K/V slots per token
    slot, each of max_cond_len rows in every AttnBlock: about 30 MB per slot on the default model at max_cond_len 132 (44
    AttnBlocks x 132 rows x 2 x 1280 fp16), so max_prompt_regions x max_batch such slots in all.  At 0 the engine allocates
    what it does without regional prompts.  ``max_guidance_prompts`` (0 .. 7): the guidance prompts a request may carry, with K/V
    slots reserved the same way: max_guidance_prompts x max_batch slots of about 30 MB each on the default model at max_cond_len
    132 (about 1.9 GB per prompt at max_batch 64).  At 0 the engine allocates what it does without guidance prompts."""

    def __init__(self, model: Paella, latent_hw=(32, 32), max_batch: int = 64, max_cond_len: int = 140,
                 unconditional_inputs: Optional[Dict[str, torch.Tensor]] = None, vqmodel=None, max_prompt_regions: int = 0,
                 max_guidance_prompts: int = 0):
        self.model, self.vqmodel = model, vqmodel
        self.H, self.W = int(latent_hw[0]), int(latent_hw[1])
        self.max_batch, self.s_max = int(max_batch), int(max_cond_len)
        if not 1 <= self.max_batch <= 65535:
            raise ValueError(f"max_batch={max_batch}: expected 1 .. 65535")
        if isinstance(max_prompt_regions, bool) or not isinstance(max_prompt_regions, int) \
                or not 0 <= max_prompt_regions <= ops.MAX_PROMPT_REGIONS:
            raise ValueError(f"max_prompt_regions={max_prompt_regions!r}: expected an int in 0 .. {ops.MAX_PROMPT_REGIONS}")
        self.max_regions = max_prompt_regions
        if isinstance(max_guidance_prompts, bool) or not isinstance(max_guidance_prompts, int) \
                or not 0 <= max_guidance_prompts <= ops.MAX_GUIDANCE_PROMPTS:
            raise ValueError(f"max_guidance_prompts={max_guidance_prompts!r}: expected an int in 0 .. {ops.MAX_GUIDANCE_PROMPTS}")
        self.max_terms = max_guidance_prompts
        ops.check_per_sample_numel(self.H * self.W * model.num_labels)
        self.dev = model._device()
        L = lib()
        model._ensure_packed()
        # conditional, own unconditional, the shared unconditional slot, then max_regions regional slots per token slot, then
        # max_terms guidance-prompt slots per token slot
        self.n_slots = 2 * self.max_batch + 1 + (self.max_regions + self.max_terms) * self.max_batch
        self.shared_slot = None
        # per-request attn_weights: a row per token slot, as long as the longest vector max_cond_len admits on this grid (bounded
        # for a model without AttnBlocks, where the weights have no effect)
        self.w_max = min(model.max_attn_weights((self.H, self.W), self.s_max), self.H * self.W + self.s_max)
        with torch.cuda.device(self.dev):
            self.tokens = torch.zeros(self.max_batch, self.H, self.W, dtype=torch.int64, device=self.dev)
            self.noise = torch.zeros_like(self.tokens)
            self._x = torch.empty_like(self.tokens)
            self._sampled = torch.empty_like(self.tokens)
            self.w_pool = torch.zeros(self.max_batch, self.w_max, dtype=torch.float32, device=self.dev)
            self.w_len = torch.zeros(self.max_batch, dtype=torch.int32, device=self.dev)
            # per-request regions: source tokens and region (True = generated) by token slot
            self.src = torch.zeros_like(self.tokens)
            self.region = torch.ones(self.max_batch, self.H, self.W, dtype=torch.bool, device=self.dev)
            self._neg_t = torch.full((self.max_batch,), -1.0, dtype=torch.float32, device=self.dev)   # composite-only t
            if self.max_regions:
                # per-request regional prompts by token slot: token masks (all bit 0 for a plain request) and region slots
                self.prompt_mask = torch.ones(self.max_batch, self.H, self.W, dtype=torch.uint8, device=self.dev)
                self.region_slot = torch.full((self.max_batch, self.max_regions), -1, dtype=torch.int32, device=self.dev)
            # zero-filled: K/V rows past a slot's kv_len are never attended to, but must be finite (see prepare_conditioning)
            self.cache = ConditioningCache(
                torch.zeros(L.pb200_paella_cond_cache_bytes(model._handle, self.n_slots, self.s_max), dtype=torch.uint8,
                            device=self.dev), self.n_slots, self.s_max, self.n_slots, None)
            model._ws(L.pb200_paella_workspace_bytes(model._handle, (2 + self.max_terms) * self.max_batch, self.H, self.W, self.s_max))
            # a request with a LoRA adapter projects these under its adapter into its own unconditional slot
            self._uncond_inputs = unconditional_inputs
            if unconditional_inputs is not None:
                self._check_cond("unconditional_inputs", unconditional_inputs)
                self.shared_slot = 2 * self.max_batch
                with torch.inference_mode():
                    model.write_conditioning(self.cache, self.shared_slot, unconditional_inputs, (self.H, self.W))
        self.map_acc: Optional[torch.Tensor] = None      # attention maps: [max_batch, max_cond_len, positions], on first use
        self._free = list(range(self.max_batch))
        self._queue: collections.deque = collections.deque()
        self._active: List[Request] = []
        self._gens = set()

    @property
    def busy(self) -> bool:
        return bool(self._active or self._queue)

    def _check_cond(self, name, inputs):
        if not isinstance(inputs, dict) or inputs.get("byt5") is None:
            raise ValueError(f"{name}: a dict with 'byt5' (and optionally 'clip', 'clip_image') is required")
        if inputs["byt5"].dim() != 3 or inputs["byt5"].shape[0] != 1:
            raise ValueError(f"{name}: byt5 of shape {list(inputs['byt5'].shape)}; a request has batch 1")
        n = self.model.conditioning_seq_len(inputs)
        if n > self.s_max:
            raise ValueError(f"{name}: conditioning of {n} rows exceeds max_cond_len={self.s_max}")

    def submit(self, model_inputs, unconditional_inputs=None, *, generator=None, steps=12, renoise_steps=None,
               temperature=(0.7, 0.3), cfg=(8.0, 8.0), t_start=1.0, t_end=0.0, sampling_conditional_steps=None, init_x=None,
               decode=False, attn_weights=None, keep_intermediates=False, region=None, mode="multinomial",
               sampling_quant_steps=None, top_k=None, top_p=None, tiling=None, prompt_regions=None, guidance_prompts=None,
               attention_maps=False, attention_source=None, lora=None, pag=None, confidence_renoise=None) -> Request:
        """Queue one request: the arguments of ``sample_distributed`` with batch 1, plus its own CUDA generator, which no other
        request in flight may use.  Raises ValueError, before anything is enqueued and before any generator advances, for a
        missing or wrong generator, conditioning longer than max_cond_len, an init_x of the wrong shape, a temperature <= 0,
        steps < 1, or an ``attn_weights`` that is not a finite 1-D CPU float tensor at most as long as the smallest key count
        the request sees in an AttnBlock, or a ``region`` that is not a bool [1, H, W] tensor on the CPU or the model's device
        or comes without init_x, a ``mode`` other than 'multinomial', 'argmax' or 'quant', a ``sampling_quant_steps`` that is not
        None or an int >= 0, or a request that would use 'quant' on an engine without vqmodel.  ``attn_weights`` weights the
        request's conditional forward as in sample_notebook; ``keep_intermediates`` collects sample_notebook's second value in
        ``req.intermediates``; ``region`` inpaints or outpaints init_x as in sample_distributed; ``mode`` and
        ``sampling_quant_steps`` choose each step's sampling mode as in sample_notebook (step k uses 'quant' if
        k >= sampling_quant_steps, ``mode`` otherwise; 'quant' reads the codebook of the engine's vqmodel).  ``top_k`` (None or
        an int >= 0) and ``top_p`` (None or a float in (0, 1]) truncate the request's multinomial steps as in sample_notebook;
        ValueError for any other value.  ``tiling`` (None, 'none', 'x', 'y' or 'xy') tiles the request as in sample_notebook, and
        with ``decode=True`` its decode; ValueError for any other value.  ``prompt_regions`` (None or a list of at most
        max_prompt_regions (inputs, region) pairs: a batch-1 conditioning dict of at most max_cond_len rows and a bool [H, W]
        region) gives the request regional prompts as in sample_notebook; ValueError for any other value, and with
        ``attn_weights``.  ``guidance_prompts`` (None or a list of at most max_guidance_prompts (inputs, weight) pairs: a batch-1
        conditioning dict of at most max_cond_len rows and a finite real weight) mixes further prompts into a guided request's
        guidance as in sample_notebook; ValueError for any other value, and on a request without cfg.  ``attention_maps=True`` sets
        ``req.attention_maps`` at retirement (module docstring); ValueError for a flag that is not a bool and with
        ``prompt_regions``.  ``attention_source=(src, k)`` makes the request a prompt-to-prompt edit of ``src`` (module
        docstring): ``src`` must be a request of this engine that is still queued and not itself an edit, neither may have
        ``prompt_regions``, both need the same conditioning length, ``steps``, ``renoise_steps`` and ``sampling_conditional_steps``,
        k is an int in 0 .. steps, and the source with all its edits must fit in max_batch; ValueError otherwise.  Give the edit a
        generator seeded like its source's.  ``lora`` (None, an adapter or (adapter, scale)) runs the request under a LoRA adapter
        as in sample_notebook, its conditional, unconditional, regional and guidance-prompt K/V included: a request with an adapter
        and no negative prompt of its own gets its own unconditional slot, into which the engine-wide unconditional inputs are
        projected under its adapter.  ValueError for a bad entry or scale and an adapter of another configuration or device.  The
        request holds its adapter until it retires.  ``pag`` (None, a scale s or (s, blocks)) adds perturbed-attention guidance
        as in sample_notebook: on the request's steps before sampling_conditional_steps, one more denoiser row, its perturbed
        forward, joins its mix (guided or not); it reads the request's conditional slot, weight row, wrap byte and adapter.
        ValueError for a bad entry (ops.pag_table), with ``prompt_regions``, and on an edit or a source.  The engine allocates
        nothing for PAG until a request uses it (then one empty row of its weight pool).  ``confidence_renoise`` (None or a choice
        temperature tau, a finite float >= 0) renoises the request's least likely tokens as in sample_notebook; ValueError for any
        other value and for a latent grid larger than the selection kernel takes (ops.confidence_table).  The request's draws
        start when it is admitted."""
        attention_maps = ops.check_attention_maps(attention_maps, prompt_regions)
        if not isinstance(generator, torch.Generator) or generator.device.type != "cuda":
            raise ValueError(f"generator: one CUDA torch.Generator per request is required (got {type(generator).__name__})")
        g_idx = generator.device.index if generator.device.index is not None else torch.cuda.current_device()
        if g_idx != self.dev.index:
            raise ValueError(f"generator is on cuda:{g_idx}, the model on {self.dev}")
        if id(generator) in self._gens:
            raise ValueError("generator is already used by a request in flight")
        if not isinstance(steps, int) or steps < 1:
            raise ValueError(f"steps={steps!r}: expected an int >= 1")
        for name, v in (("top_k", top_k), ("top_p", top_p)):
            if torch.is_tensor(v):
                raise ValueError(f"{name}: a request takes one value (got a tensor)")
        trunc = ops.truncation_table(top_k, top_p, 1, self.model.num_labels)
        if isinstance(tiling, (list, tuple)):
            raise ValueError("tiling: a request takes one value (got a list)")
        wrap = ops.tiling_codes(tiling, 1)[0]
        renoise_steps = steps - 1 if renoise_steps is None else int(renoise_steps)
        cond_steps = steps if sampling_conditional_steps is None else int(sampling_conditional_steps)
        self._check_cond("model_inputs", model_inputs)
        if unconditional_inputs is not None:
            self._check_cond("unconditional_inputs", unconditional_inputs)
        elif cfg is not None and self.shared_slot is None:
            raise ValueError("cfg is set but there are no unconditional inputs (per request or engine-wide)")
        if init_x is not None and tuple(init_x.shape) != (1, self.H, self.W):
            raise ValueError(f"init_x of shape {list(init_x.shape)}; expected [1, {self.H}, {self.W}]")
        U.check_region(region, init_x, (1, self.H, self.W), self.dev)
        if decode and self.vqmodel is None:
            raise ValueError("decode=True needs the engine's vqmodel")
        mode = ops.check_mode("mode", mode)
        sampling_quant_steps = ops.check_quant_steps("sampling_quant_steps", sampling_quant_steps)
        if self.vqmodel is None and any(ops.mode_at(mode, sampling_quant_steps, k) == "quant" for k in range(steps)):
            raise ValueError("mode 'quant' (or sampling_quant_steps) needs the VQGAN codebook: build the engine with vqmodel=...")
        regions = None
        if prompt_regions is not None:
            if not isinstance(prompt_regions, (list, tuple)) or len(prompt_regions) > self.max_regions:
                raise ValueError(f"prompt_regions: at most max_prompt_regions={self.max_regions} (inputs, region) pairs per request")
            regions = ops.regional_table([prompt_regions], 1, (self.H, self.W), self.dev)
            ops.check_regions_unweighted(regions, attn_weights)
            if regions is not None:
                for k, inputs in enumerate(regions[1][0]):
                    self._check_cond(f"prompt_regions[{k}]", inputs)
                regions = (regions[0][0], regions[1][0])
        terms = None
        if guidance_prompts is not None:
            if not isinstance(guidance_prompts, (list, tuple)) or len(guidance_prompts) > self.max_terms:
                raise ValueError(f"guidance_prompts: at most max_guidance_prompts={self.max_terms} (inputs, weight) pairs per request")
            table = ops.guidance_table([guidance_prompts], 1)
            if table is not None:
                terms = table[0]
                for j, (inputs, _) in enumerate(terms):
                    self._check_cond(f"guidance_prompts[{j}]", inputs)
                if cfg is None:
                    raise ValueError("guidance_prompts need a guided request (cfg is None)")
        if attn_weights is not None:
            n_keys = self.model.max_attn_weights((self.H, self.W), self.model.conditioning_seq_len(model_inputs))
            attn_weights = ops.check_attn_weight_vector("attn_weights", attn_weights, min(n_keys, self.w_max))
        if isinstance(lora, list):
            raise ValueError("lora: a request takes one entry (got a list)")
        lora = ops.lora_entries(ops.lora_table(lora, 1, self.model), 1)[0]
        if attention_source is not None:
            self._check_attention_source(attention_source, model_inputs, steps, renoise_steps, cond_steps, prompt_regions, lora)
        pag_e = None
        if pag is not None:
            if isinstance(pag, list):
                raise ValueError("pag: a request takes one entry (got a list)")
            pag_t = ops.pag_table([pag], 1, self.model.n_attn_blocks, self.model.pag_default_blocks())
            if pag_t is not None:
                if prompt_regions:
                    raise ValueError("pag: perturbed-attention guidance on a request with prompt_regions is not supported")
                if attention_source is not None:
                    raise ValueError("pag: perturbed-attention guidance on a prompt-to-prompt edit is not supported")
                pag_e = (pag_t[0][0], int(pag_t[1][0]))
        if isinstance(confidence_renoise, (list, tuple)):
            raise ValueError("confidence_renoise: a request takes one value (got a list)")
        conf = ops.confidence_table(confidence_renoise, 1, self.H * self.W)
        cfgs = U._cfg_schedule(cfg, 1, steps)
        params, r = U.sampling_schedule(1, steps, temperature, cfgs, t_start, t_end, torch.is_tensor(cfg), always=True)
        mix_coef = None
        n_mix = min(steps, cond_steps)
        s = pag_e[0] if pag_e is not None else 0.0
        if terms is not None or (pag_e is not None and cfgs is not None):
            # the guided steps' mix coefficients; their params rows become (1, 0, 1/T): f*1 + u*0 = f
            step_cfg = cfgs[0] if torch.is_tensor(cfg) else cfgs
            ws = [w for _, w in terms] if terms is not None else []
            mix_coef = torch.tensor([ops.guidance_coefficients(step_cfg[i], ws, s) for i in range(n_mix)],
                                    dtype=torch.float32).view(n_mix, 2 + len(ws) + (pag_e is not None))
            params[:n_mix, 0, 0] = 1.0
            params[:n_mix, 0, 1] = 0.0
        elif pag_e is not None:    # unguided: l_c + s (l_c - l_p)
            mix_coef = torch.tensor([ops.guidance_coefficients(None, [], s)] * n_mix, dtype=torch.float32).view(n_mix, 2)
        req = Request(steps, renoise_steps, cond_steps, cfgs is not None, params[:, 0], r[:, 0], generator, model_inputs,
                      unconditional_inputs, init_x, bool(decode), attn_weights, bool(keep_intermediates), region, mode,
                      sampling_quant_steps, *((int(trunc[0][0]), float(trunc[1][0])) if trunc is not None else (0, 1.0)), wrap, regions,
                      terms, mix_coef, attention_maps, self.model.conditioning_seq_len(model_inputs), attention_source, lora, pag_e,
                      float(conf[0]) if conf is not None else -1.0)
        if attention_source is not None:
            attention_source[0].edits.append(req)
        self._gens.add(id(generator))
        self._queue.append(req)
        return req

    def _check_attention_source(self, attention_source, model_inputs, steps, renoise_steps, cond_steps, prompt_regions, lora=None):
        """submit's rules for ``attention_source`` (ValueError)."""
        if not isinstance(attention_source, (list, tuple)) or len(attention_source) != 2 or not isinstance(attention_source[0], Request) \
                or isinstance(attention_source[1], bool) or not isinstance(attention_source[1], int):
            raise ValueError(f"attention_source: expected a (Request, int steps) pair (got {attention_source!r})")
        src, k = attention_source
        if not any(q is src for q in self._queue):
            raise ValueError("attention_source: the source must be a request of this engine that is still queued")
        if src.inj_src is not None:
            raise ValueError("attention_source: the source is itself an edit (no chains)")
        if src.regional or prompt_regions:
            raise ValueError("attention_source: prompt_regions on an edit or on its source are not supported")
        if src.pag is not None:
            raise ValueError("attention_source: perturbed-attention guidance on the source is not supported")
        if src.maps_len != self.model.conditioning_seq_len(model_inputs):
            raise ValueError(f"attention_source: the source's conditioning has {src.maps_len} rows, the edit's "
                             f"{self.model.conditioning_seq_len(model_inputs)}")
        if (src.steps, src.renoise_steps, src.cond_steps) != (steps, renoise_steps, cond_steps):
            raise ValueError("attention_source: the edit needs its source's steps, renoise_steps and sampling_conditional_steps")
        if not 0 <= k <= steps:
            raise ValueError(f"attention_source: {k} injected steps; expected 0..{steps}")
        if len(src.edits) + 2 > self.max_batch:
            raise ValueError(f"attention_source: a source and its {len(src.edits) + 1} edits exceed max_batch={self.max_batch}")
        if len(ops.distinct_adapters([q.lora for q in [src] + src.edits] + [lora])) > ops.MAX_LORA_ADAPTERS:
            raise ValueError(f"attention_source: a source and its edits on more than {ops.MAX_LORA_ADAPTERS} distinct LoRA adapters "
                             "cannot be admitted together")

    def _admit(self):
        new = admit_from_queue(self._queue, len(self._free), self._active)
        for q in new:
            q.slot = self._free.pop(0)
            # an adapter is part of the model: a request with one never reads the shared unconditional slot
            if q.uncond is None and q.lora is not None and q.guided and self.shared_slot is not None:
                q.uncond = self._uncond_inputs
            q.uncond_slot = self.max_batch + q.slot if q.uncond is not None else self.shared_slot
        if not new:
            return
        if any(q.pag is not None for q in new) and self.w_pool.shape[0] == self.max_batch:
            # perturbed-attention guidance: one weight row of length 0 (row max_batch) for the unconditional and term rows of a
            # perturbing step, whose w_row covers every row
            self.w_pool = torch.cat([self.w_pool, torch.zeros(1, self.w_max, dtype=torch.float32, device=self.dev)])
            self.w_len = torch.cat([self.w_len, torch.zeros(1, dtype=torch.int32, device=self.dev)])
        m = self.model
        hw = self.H * self.W
        table = ops.philox_table([q.generator for q in new], hw, self.dev)
        # one copy: the slots, then each request's weight row and length, written into the pool (a request without weights
        # gets length 0, so a reused slot never reads the entries of its previous request), then each request's region row
        # (all True without a region, for the same reason) and the source tokens that come from the CPU
        w_rows, w_lens = ops.attn_weights_table([q.attn_weights for q in new], len(new), [self.w_max] * len(new))
        w_rows = torch.nn.functional.pad(w_rows, (0, self.w_max - w_rows.shape[1]))
        n = len(new)
        regions = torch.ones(n, self.H, self.W, dtype=torch.bool)
        for j, q in enumerate(new):
            if q.has_region and q.region.device.type == "cpu":
                regions[j] = q.region[0]
        host_src = [q for q in new if q.has_region and q.init_x.device.type == "cpu"]
        src_row = {id(q): j for j, q in enumerate(host_src)}
        srcs = torch.cat([q.init_x.to(torch.int64) for q in host_src]) if host_src else torch.zeros(0, dtype=torch.int64)
        # regional prompts: each request's token masks (all bit 0 without regions) and the K/V slots reserved for its token slot
        R = self.max_regions
        masks = torch.ones(n, self.H, self.W, dtype=torch.uint8)
        rslots = torch.full((n, R), -1, dtype=torch.int32)
        region_writes = []
        for j, q in enumerate(new):
            if q.regional:
                masks[j] = q.regions[0]
                for k, inputs in enumerate(q.regions[1]):
                    rslots[j, k] = self._region_slot(q.slot, k)
                    region_writes.append((self._region_slot(q.slot, k), inputs, q.lora))
        slots, w_lens_d, w_rows_d, regions_d, srcs_d, *regional_d = ops.to_device_packed(
            [torch.tensor([q.slot for q in new], dtype=torch.int32), w_lens, w_rows, regions, srcs] + ([masks, rslots] if R else []),
            self.dev)
        self.w_len.index_copy_(0, slots.long(), w_lens_d)
        self.w_pool.index_copy_(0, slots.long(), w_rows_d)
        self.region.index_copy_(0, slots.long(), regions_d)
        if R:
            self.prompt_mask.index_copy_(0, slots.long(), regional_d[0])
            self.region_slot.index_copy_(0, slots.long(), regional_d[1])
        if any(q.want_maps for q in new):
            if self.map_acc is None:
                self.map_acc = m.map_accumulator(self.max_batch, self.s_max, (self.H, self.W))
            for q in new:
                if q.want_maps:
                    self.map_acc[q.slot].zero_()
        ops.randint_per_sample(self.noise, m.num_labels, table, slot=slots, batch=n)
        for q in new:
            s = q.slot
            if q.has_region:             # tokens = where(region, noise, init_x)
                if q.region.device.type != "cpu":
                    self.region[s].copy_(q.region[0], non_blocking=True)
                self.src[s].copy_(srcs_d[src_row[id(q)]] if id(q) in src_row else q.init_x[0], non_blocking=True)
                ops.composite(self.noise[s:s + 1], self.src[s:s + 1], self.region[s:s + 1], self._neg_t[:1], out=self.tokens[s:s + 1])
            else:
                src = self.noise[s] if q.init_x is None else q.init_x[0]
                self.tokens[s].copy_(src, non_blocking=True)
        # the conditional and own unconditional K/V of the admitted requests: one projection per run of contiguous slots with
        # one sequence layout (the rows equal per-request projections bit for bit: the conditioning path has no statistic
        # that spans rows)
        for q in new:
            q.term_slot = [self._term_slot(q.slot, j) for j in range(q.n_terms)]
        term_writes = [(s, inputs, q.lora) for q in new for s, (inputs, _) in zip(q.term_slot, q.terms or [])]
        writes = [(q.slot, q.inputs, q.lora) for q in new] + [(q.uncond_slot, q.uncond, q.lora) for q in new if q.uncond is not None] \
            + region_writes + term_writes
        for run in admission_runs([(slot, cond_layout(x)) for slot, x, _ in writes]):
            entries = [writes[i][2] for i in run]
            m.write_conditioning(self.cache, writes[run[0]][0], _cat_inputs([writes[i][1] for i in run], self.dev), (self.H, self.W),
                                 lora=entries if any(e is not None for e in entries) else None)
        for q in new:
            q.inputs = q.uncond = q.init_x = q.region = q.regions = q.terms = None
        self._active += new

    def _region_slot(self, token_slot: int, k: int) -> int:
        """The K/V slot of regional prompt k of the request in ``token_slot``."""
        return 2 * self.max_batch + 1 + token_slot * self.max_regions + k

    def _term_slot(self, token_slot: int, j: int) -> int:
        """The K/V slot of guidance prompt j of the request in ``token_slot``."""
        return 2 * self.max_batch + 1 + self.max_regions * self.max_batch + token_slot * self.max_terms + j

    def step(self) -> List[Request]:
        """Admit what fits, advance every active request by one of its own steps, and return the requests that finished
        (in admission order), their ``result`` set.  No host synchronisation."""
        with torch.inference_mode(), torch.cuda.device(self.dev):
            self._admit()
            if not self._active:
                return []
            plan = build_step_plan(self._active, self.max_batch)
            m, dev, H, W = self.model, self.dev, self.H, self.W
            Bc, n_pairs = len(plan.order), plan.n_pairs
            hw = H * W
            draw, renoise = [], []
            for q, dr, rn in zip(plan.order, plan.draws, plan.renoise):     # per request: the sampler's draw, then the mask draw
                draw += ops.philox_values([q.generator], hw * m.num_labels, dev) if dr else [0, 0]
                renoise += ops.philox_values([q.generator], hw, dev) if rn else [0, 0]
            mixed = not all(plan.draws)
            host, lay = step_host_table(plan, draw, renoise)
            buf = ops.to_device_async(host, dev)                 # the step's one host-to-device copy
            draw_d, renoise_d = buf[:2 * Bc].view(Bc, 2), buf[2 * Bc:4 * Bc].view(Bc, 2)
            parts = {"f32": buf[lay["f32"][1]:lay["f32"][1] + lay["f32"][2]].view(torch.float32),
                     "i32": buf[lay["i32"][1]:lay["i32"][1] + lay["i32"][2]].view(torch.int32),
                     "u8": buf[lay["u8"][1]:lay["u8"][1] + lay["u8"][2]].view(torch.uint8)}

            def part(name):
                dt, o, n = lay[name]
                return parts[dt][o:o + n]
            r_d, params_d, t_next_d = part("r"), part("params").view(Bc, 3), part("t_next")
            row_slot_d, kv_slot_d, modes_d = part("row_slot"), part("kv_slot"), part("modes")
            trunc_d = (part("top_k"), part("top_p")) if plan.truncates else None
            wrap_d = part("wrap") if plan.wraps else None
            n_tail = plan.tail.numel() if plan.composed else n_pairs
            tail = dict(tail_src=part("tail")) if plan.composed else dict(n_pairs=n_pairs)
            if plan.maps:       # row b accumulates into its token slot's maps
                tail["maps"] = (part("map_row"), Bc, self.map_acc)
            if plan.injects:    # row b replays the attention of row inj_src[b]
                tail["inject"] = part("inj_src")
            if plan.loras:      # row b runs under adapter lora_id[b] (its tail rows under their source's)
                tail["lora"] = (ops.lora_structs(plan.adapters), len(plan.adapters), part("lora_id"), part("lora_scale"))
            if plan.perturbed:  # the perturbed rows' AttnBlock masks
                tail["perturb"] = buf[lay["pag"][1]:lay["pag"][1] + lay["pag"][2]]

            x = ops.gather_rows(self.tokens, row_slot_d, self._x[:Bc])
            cond = ConditioningCache(self.cache.cache, Bc + n_tail, self.s_max, self.n_slots, kv_slot_d)
            # row b reads the regional prompts of its token slot
            regional = (self.prompt_mask, self.region_slot, row_slot_d) if any(q.regional for q in plan.order) else None
            if any(q.attn_weights is not None for q in plan.order) and plan.perturbed:
                # every row reads its weight row: a perturbed row its request's, the unconditional and term rows the empty one
                feats = m.features(x, r_d, cond, self.w_pool, Bc + n_tail, w_len=self.w_len, w_row=part("w_row"), wrap=wrap_d,
                                   regional=regional, **tail)
            elif any(q.attn_weights is not None for q in plan.order):       # row b reads the weights of its token slot
                feats = m.features(x, r_d, cond, self.w_pool, Bc, w_len=self.w_len, w_row=row_slot_d, wrap=wrap_d, regional=regional,
                                   **tail)
            else:
                feats = m.features(x, r_d, cond, wrap=wrap_d, regional=regional, **tail)
            if plan.composed:       # each composed row becomes its guided mix, sampled with (1, 0, 1/T)
                J2 = plan.mix_rows.shape[1]
                m.guidance_mix(feats, hw, part("mix_rows").view(-1, J2), part("mix_coef").view(-1, J2))
            if mixed:       # argmax and quant rows through the logits path, the multinomial rows in one fused-sampler launch
                sampled = m.sample_tokens_modes(feats, Bc, n_pairs, H, W, params_d, draw_d, plan.modes, modes_d, self._codebook(),
                                                out=self._sampled[:Bc], trunc=trunc_d)
            else:
                sampled = m.sample_tokens_pairs(feats, Bc, n_pairs, H, W, params_d, draw_d, out=self._sampled[:Bc], trunc=trunc_d)
            for i, q in enumerate(plan.order):
                if q.intermediates is not None:
                    s = q.slot
                    q.intermediates.append(ops.composite(sampled[i:i + 1], self.src[s:s + 1], self.region[s:s + 1], self._neg_t[:1])
                                           if q.has_region else sampled[i:i + 1].clone())
            # every row back into its slot, renoised or not; with a region in the batch, each row's source tokens outside it
            regions = any(q.has_region for q in plan.order)
            if plan.confident:      # the rows' confidence from the operand the step's sampler read
                logp = m.token_logprob(feats, Bc, n_pairs, hw, params_d, sampled)
                ops.renoise_confidence_per_sample(sampled, t_next_d, part("tau"), logp, self.noise, renoise_d, self.tokens, slot=row_slot_d,
                                                  src=self.src if regions else None, region=self.region if regions else None)
            else:
                ops.add_noise_per_sample(sampled, t_next_d, self.noise, m.num_labels, renoise_d, self.tokens, slot=row_slot_d,
                                         src=self.src if regions else None, region=self.region if regions else None)
            for q, rn in zip(plan.order, plan.renoise):
                if q.intermediates is not None and rn:
                    q.intermediates.append(self.tokens[q.slot:q.slot + 1].clone())

            for q in plan.order:
                q.k += 1
            done = [q for q in self._active if q.k == q.steps]
            if not done:
                return []
            dec = [q for q in done if q.decode]
            if dec:
                tiling = [("none", "x", "y", "xy")[q.wrap] for q in dec]
                imgs = self.vqmodel.decode_indices_u8(torch.cat([self.tokens[q.slot:q.slot + 1] for q in dec]), tiling)
                for i, q in enumerate(dec):
                    q.result = imgs[i:i + 1]
            for q in done:
                if q.want_maps:
                    q.attention_maps = m.finalize_attention_maps(self.map_acc[q.slot:q.slot + 1], (H, W), q.maps_len, q.steps)[0]
                if not q.decode:
                    q.result = self.tokens[q.slot:q.slot + 1].clone()
                self._free.append(q.slot)
                self._gens.discard(id(q.generator))
                q.lora = None
            self._free.sort()
            self._active = [q for q in self._active if q.k < q.steps]
            return done

    def _codebook(self) -> Optional[torch.Tensor]:
        return self.vqmodel.vquantizer.codebook.weight.data if self.vqmodel is not None else None

    def run_until_idle(self) -> List[Request]:
        """Step until nothing is active or queued; returns every request finished on the way, in finishing order."""
        out = []
        while self.busy:
            out += self.step()
        return out
