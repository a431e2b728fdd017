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
region=region)``: a step in argmax or quant mode draws nothing from ``g`` (only its mask draw, if it renoises).

Each step orders its batch with the guided requests first: rows [0, n_pairs) are guided, [n_pairs, Bc) are not, and the
unconditional rows of the guided ones follow as [Bc, Bc + n_pairs) (Paella.features with ``n_pairs``).  Per step the host
builds one table (noise levels, (cfg, 1 - cfg, 1/T), renoise targets, Philox (seed, offset) pairs, row -> slot maps) and
sends it to the device with one asynchronous copy; the step itself is a gather of the rows from the token pool, the forward,
one fused-sampler launch and one per-sample add-noise launch that writes every row back into its slot.  A step whose rows are
in several sampling modes adds each row's mode to the table: the fused sampler skips the argmax and quant rows, which then go
through the out_mapper GEMM to logits (a bounded number of samples at a time) and the argmax or quant kernel, one call per mode
(Paella.sample_tokens_modes).  The host knows which
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
                 region: Optional[torch.Tensor] = None, mode: str = "multinomial", quant_steps: Optional[int] = None):
        self.steps, self.renoise_steps, self.cond_steps, self.guided = steps, renoise_steps, cond_steps, guided
        self.params, self.r = params, r          # CPU float32 [steps, 3] and [steps + 1]: rows of utils.sampling_schedule
        self.generator, self.inputs, self.uncond, self.init_x, self.decode = generator, inputs, uncond, init_x, decode
        self.attn_weights = attn_weights         # CPU float32 [n] or None
        self.region = region                     # bool [1, H, W] or None, until admission
        self.has_region = region is not None
        self.mode, self.quant_steps = mode, quant_steps      # sampling mode, and the step from which 'quant' is used (or None)
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
    """The host tables of one step (CPU tensors), rows in batch order: guided requests first."""

    def __init__(self, order: List[Request]):
        self.order = order
        self.n_pairs = sum(1 for q in order if q.guided and q.k < q.cond_steps)
        self.r = torch.stack([q.r[q.k] for q in order])
        self.params = torch.stack([q.params[q.k] for q in order])
        self.renoise = [q.k < q.renoise_steps for q in order]
        self.modes = [q.mode_at(q.k) for q in order]
        self.draws = [md == "multinomial" for md in self.modes]     # only multinomial rows draw the sampler's exponentials
        # a row that does not renoise keeps its tokens (t < 0 never passes the mask test)
        self.t_next = torch.stack([q.r[q.k + 1] if rn else torch.tensor(-1.0) for q, rn in zip(order, self.renoise)])
        self.row_slot = torch.tensor([q.slot for q in order], dtype=torch.int32)
        self.kv_slot = torch.tensor([q.slot for q in order] + [q.uncond_slot for q in order[:self.n_pairs]], dtype=torch.int32)


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


def build_step_plan(active: List[Request]) -> StepPlan:
    """Order the active requests for one step -- guided this step first, each group in admission order -- and build the
    step's tables from each request's own schedule rows at its own step index."""
    guided = [q for q in active if q.guided and q.k < q.cond_steps]
    return StepPlan(guided + [q for q in active if not (q.guided and q.k < q.cond_steps)])


class SamplingEngine:
    """Step-level batcher over one Paella model and one latent grid (module docstring).

    ``max_batch`` requests are in flight at most; later ones queue and are admitted FIFO at step boundaries.  Conditioning of
    up to ``max_cond_len`` rows.  ``unconditional_inputs`` (batch 1) is projected once and used by every guided request that
    brings no negative prompt of its own.  ``vqmodel`` decodes the requests submitted with ``decode=True``."""

    def __init__(self, model: Paella, latent_hw=(32, 32), max_batch: int = 64, max_cond_len: int = 140,
                 unconditional_inputs: Optional[Dict[str, torch.Tensor]] = None, vqmodel=None):
        self.model, self.vqmodel = model, vqmodel
        self.H, self.W = int(latent_hw[0]), int(latent_hw[1])
        self.max_batch, self.s_max = int(max_batch), int(max_cond_len)
        if not 1 <= self.max_batch <= 65535:
            raise ValueError(f"max_batch={max_batch}: expected 1 .. 65535")
        ops.check_per_sample_numel(self.H * self.W * model.num_labels)
        self.dev = model._device()
        L = lib()
        model._ensure_packed()
        self.n_slots = 2 * self.max_batch + 1        # conditional, own unconditional, and the shared unconditional slot
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
            # zero-filled: K/V rows past a slot's kv_len are never attended to, but must be finite (see prepare_conditioning)
            self.cache = ConditioningCache(
                torch.zeros(L.pb200_paella_cond_cache_bytes(model._handle, self.n_slots, self.s_max), dtype=torch.uint8,
                            device=self.dev), self.n_slots, self.s_max, self.n_slots, None)
            model._ws(L.pb200_paella_workspace_bytes(model._handle, 2 * self.max_batch, self.H, self.W, self.s_max))
            if unconditional_inputs is not None:
                self._check_cond("unconditional_inputs", unconditional_inputs)
                self.shared_slot = 2 * self.max_batch
                with torch.inference_mode():
                    model.write_conditioning(self.cache, self.shared_slot, unconditional_inputs, (self.H, self.W))
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
               sampling_quant_steps=None) -> Request:
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
        k >= sampling_quant_steps, ``mode`` otherwise; 'quant' reads the codebook of the engine's vqmodel).  The request's draws
        start when it is admitted."""
        if not isinstance(generator, torch.Generator) or generator.device.type != "cuda":
            raise ValueError(f"generator: one CUDA torch.Generator per request is required (got {type(generator).__name__})")
        g_idx = generator.device.index if generator.device.index is not None else torch.cuda.current_device()
        if g_idx != self.dev.index:
            raise ValueError(f"generator is on cuda:{g_idx}, the model on {self.dev}")
        if id(generator) in self._gens:
            raise ValueError("generator is already used by a request in flight")
        if not isinstance(steps, int) or steps < 1:
            raise ValueError(f"steps={steps!r}: expected an int >= 1")
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
        if attn_weights is not None:
            n_keys = self.model.max_attn_weights((self.H, self.W), self.model.conditioning_seq_len(model_inputs))
            attn_weights = ops.check_attn_weight_vector("attn_weights", attn_weights, min(n_keys, self.w_max))
        cfgs = U._cfg_schedule(cfg, 1, steps)
        params, r = U.sampling_schedule(1, steps, temperature, cfgs, t_start, t_end, torch.is_tensor(cfg), always=True)
        req = Request(steps, renoise_steps, cond_steps, cfgs is not None, params[:, 0], r[:, 0], generator, model_inputs,
                      unconditional_inputs, init_x, bool(decode), attn_weights, bool(keep_intermediates), region, mode,
                      sampling_quant_steps)
        self._gens.add(id(generator))
        self._queue.append(req)
        return req

    def _admit(self):
        new = []
        while self._queue and self._free:
            q = self._queue.popleft()
            q.slot = self._free.pop(0)
            q.uncond_slot = self.max_batch + q.slot if q.uncond is not None else self.shared_slot
            new.append(q)
        if not new:
            return
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
        slots, w_lens_d, w_rows_d, regions_d, srcs_d = ops.to_device_packed(
            [torch.tensor([q.slot for q in new], dtype=torch.int32), w_lens, w_rows, regions, srcs], self.dev)
        self.w_len.index_copy_(0, slots.long(), w_lens_d)
        self.w_pool.index_copy_(0, slots.long(), w_rows_d)
        self.region.index_copy_(0, slots.long(), regions_d)
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
        writes = [(q.slot, q.inputs) for q in new] + [(q.uncond_slot, q.uncond) for q in new if q.uncond is not None]
        for run in admission_runs([(slot, cond_layout(x)) for slot, x in writes]):
            m.write_conditioning(self.cache, writes[run[0]][0], _cat_inputs([writes[i][1] for i in run], self.dev), (self.H, self.W))
        for q in new:
            q.inputs = q.uncond = q.init_x = q.region = None
        self._active += new

    def step(self) -> List[Request]:
        """Admit what fits, advance every active request by one of its own steps, and return the requests that finished
        (in admission order), their ``result`` set.  No host synchronisation."""
        with torch.inference_mode(), torch.cuda.device(self.dev):
            self._admit()
            if not self._active:
                return []
            plan = build_step_plan(self._active)
            m, dev, H, W = self.model, self.dev, self.H, self.W
            Bc, n_pairs = len(plan.order), plan.n_pairs
            hw = H * W
            draw, renoise = [], []
            for q, dr, rn in zip(plan.order, plan.draws, plan.renoise):     # per request: the sampler's draw, then the mask draw
                draw += ops.philox_values([q.generator], hw * m.num_labels, dev) if dr else [0, 0]
                renoise += ops.philox_values([q.generator], hw, dev) if rn else [0, 0]
            mixed = not all(plan.draws)
            modes = ops.mode_table(plan.modes) if mixed else torch.zeros(0, dtype=torch.int32)
            f32 = torch.cat([plan.r, plan.params.view(-1), plan.t_next] + ([torch.zeros(1)] if Bc % 2 else []))
            i32 = torch.cat([plan.row_slot, plan.kv_slot, modes] + ([torch.zeros(1, dtype=torch.int32)] if (n_pairs + modes.numel()) % 2 else []))
            host = torch.cat([torch.tensor(draw + renoise, dtype=torch.int64), f32.view(torch.int64), i32.view(torch.int64)])
            buf = ops.to_device_async(host, dev)                 # the step's one host-to-device copy
            draw_d, renoise_d = buf[:2 * Bc].view(Bc, 2), buf[2 * Bc:4 * Bc].view(Bc, 2)
            f32_d = buf[4 * Bc:4 * Bc + f32.numel() // 2].view(torch.float32)
            i32_d = buf[4 * Bc + f32.numel() // 2:].view(torch.int32)
            r_d, params_d, t_next_d = f32_d[:Bc], f32_d[Bc:4 * Bc].view(Bc, 3), f32_d[4 * Bc:5 * Bc]
            row_slot_d, kv_slot_d = i32_d[:Bc], i32_d[Bc:2 * Bc + n_pairs]
            modes_d = i32_d[2 * Bc + n_pairs:2 * Bc + n_pairs + modes.numel()]

            x = ops.gather_rows(self.tokens, row_slot_d, self._x[:Bc])
            cond = ConditioningCache(self.cache.cache, Bc + n_pairs, self.s_max, self.n_slots, kv_slot_d)
            if any(q.attn_weights is not None for q in plan.order):       # row b reads the weights of its token slot
                feats = m.features(x, r_d, cond, self.w_pool, Bc, n_pairs=n_pairs, w_len=self.w_len, w_row=row_slot_d)
            else:
                feats = m.features(x, r_d, cond, n_pairs=n_pairs)
            if mixed:       # argmax and quant rows through the logits path, the multinomial rows in one fused-sampler launch
                sampled = m.sample_tokens_modes(feats, Bc, n_pairs, H, W, params_d, draw_d, plan.modes, modes_d, self._codebook(),
                                                out=self._sampled[:Bc])
            else:
                sampled = m.sample_tokens_pairs(feats, Bc, n_pairs, H, W, params_d, draw_d, out=self._sampled[:Bc])
            for i, q in enumerate(plan.order):
                if q.intermediates is not None:
                    s = q.slot
                    q.intermediates.append(ops.composite(sampled[i:i + 1], self.src[s:s + 1], self.region[s:s + 1], self._neg_t[:1])
                                           if q.has_region else sampled[i:i + 1].clone())
            # every row back into its slot, renoised or not; with a region in the batch, each row's source tokens outside it
            regions = any(q.has_region for q in plan.order)
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
                imgs = self.vqmodel.decode_indices_u8(torch.cat([self.tokens[q.slot:q.slot + 1] for q in dec]))
                for i, q in enumerate(dec):
                    q.result = imgs[i:i + 1]
            for q in done:
                if not q.decode:
                    q.result = self.tokens[q.slot:q.slot + 1].clone()
                self._free.append(q.slot)
                self._gens.discard(id(q.generator))
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
