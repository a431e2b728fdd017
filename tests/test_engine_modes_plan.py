"""Per-request sampling modes without a device: the mode of every row of SamplingEngine's step plan (the switch to 'quant' at
``sampling_quant_steps``), which rows draw the sampler's exponentials, the generator offsets that follow from the plan, the
device mode table, and the validation of sample_notebook's per-sample ``mode`` / ``sampling_quant_steps``."""
import random

import pytest
import torch

from paella_b200 import ops
from paella_b200 import utils as U
from paella_b200._lib import lib
from paella_b200.engine import Request, build_step_plan


def _request(rng, slot, mode, quant_steps, steps):
    cfg = rng.choice([None, (8.0, 8.0)])
    cfgs = U._cfg_schedule(cfg, 1, steps)
    params, r = U.sampling_schedule(1, steps, (0.7, 0.3), cfgs, 1.0, 0.0, always=True)
    renoise = rng.choice([steps - 1, 0, steps // 2])
    q = Request(steps, renoise, rng.choice([steps, steps // 2]), cfg is not None, params[:, 0], r[:, 0], mode=mode,
                quant_steps=quant_steps)
    q.slot, q.uncond_slot = slot, 99
    return q


def test_mode_at_switches_to_quant_at_sampling_quant_steps():
    q = Request(5, 4, 5, False, torch.zeros(5, 3), torch.zeros(6), mode="argmax", quant_steps=2)
    assert [q.mode_at(k) for k in range(5)] == ["argmax", "argmax", "quant", "quant", "quant"]
    q = Request(3, 2, 3, False, torch.zeros(3, 3), torch.zeros(4), mode="multinomial", quant_steps=0)
    assert [q.mode_at(k) for k in range(3)] == ["quant"] * 3
    q = Request(3, 2, 3, False, torch.zeros(3, 3), torch.zeros(4), mode="multinomial", quant_steps=None)
    assert [q.mode_at(k) for k in range(3)] == ["multinomial"] * 3
    q = Request(3, 2, 3, False, torch.zeros(3, 3), torch.zeros(4))           # the default: multinomial throughout
    assert [q.mode_at(k) for k in range(3)] == ["multinomial"] * 3
    assert ops.mode_at("argmax", 7, 6) == "argmax" and ops.mode_at("argmax", 7, 7) == "quant"


def test_step_plan_modes_draws_and_generator_offsets():
    """Run the plans of a staggered mixed load to the end, counting each request's Philox offsets the way SamplingEngine.step
    takes them; they must equal the batch-1 sample_notebook loop's (randint, then per step the exponential draw if the step is
    multinomial and the mask draw if it renoises)."""
    rng = random.Random(3)
    hw, NL = 64, 512
    inc = lib().pb200_philox_offset_increment
    for trial in range(50):
        reqs = []
        for j in range(rng.randint(1, 10)):
            steps = rng.choice([1, 2, 4, 8])
            mode = rng.choice(ops.SAMPLING_MODES)
            qs = rng.choice([None, 0, 2, 6])
            reqs.append(_request(rng, j, mode, qs, steps))
        offs = {id(q): inc(hw) for q in reqs}                   # the randint at admission
        active = list(reqs)
        while active:
            plan = build_step_plan(active)
            assert plan.modes == [q.mode_at(q.k) for q in plan.order]
            assert plan.draws == [md == "multinomial" for md in plan.modes]
            tab = ops.mode_table(plan.modes)
            Bc = len(plan.order)
            assert tab.dtype == torch.int32 and tab[:Bc].tolist() == [ops.SAMPLING_MODES.index(md) for md in plan.modes]
            lists = tab[Bc:].tolist()
            n_arg = plan.modes.count("argmax")
            assert lists[:n_arg] == [b for b, md in enumerate(plan.modes) if md == "argmax"]
            assert lists[n_arg:] == [b for b, md in enumerate(plan.modes) if md == "quant"]
            # ascending lists put the guided rows (b < n_pairs) first, as pb200_paella_resample_samples requires
            for sub in (lists[:n_arg], lists[n_arg:]):
                guided = [b < plan.n_pairs for b in sub]
                assert guided == sorted(guided, reverse=True)
            for q, dr, rn in zip(plan.order, plan.draws, plan.renoise):
                offs[id(q)] += (inc(hw * NL) if dr else 0) + (inc(hw) if rn else 0)
                q.k += 1
            active = [q for q in active if q.k < q.steps]
        for q in reqs:
            want = inc(hw)
            for i in range(q.steps):
                md = "quant" if q.quant_steps is not None and i >= q.quant_steps else q.mode
                want += (inc(hw * NL) if md == "multinomial" else 0) + (inc(hw) if i < q.renoise_steps else 0)
            assert offs[id(q)] == want


def test_sampling_modes_scalar_uniform_and_mixed():
    gens = ["g0", "g1", "g2"]          # only the list shape matters here
    assert U.sampling_modes("argmax", 2, 3, 4) is None                               # scalar: today's path
    assert U.sampling_modes(["argmax"] * 3, None, 3, 4) is None                       # all entries equal
    assert U.sampling_modes("multinomial", [1, 1, 1], 3, 4, codebook=torch.zeros(1)) is None
    t = U.sampling_modes(["multinomial", "argmax", "quant"], [None, 1, None], 3, 3, gens, codebook=torch.zeros(1))
    assert t == [["multinomial", "argmax", "quant"], ["multinomial", "quant", "quant"], ["multinomial", "quant", "quant"]]
    t = U.sampling_modes("argmax", [0, None, 2], 3, 3, gens, codebook=torch.zeros(1))
    assert t == [["quant", "argmax", "argmax"], ["quant", "argmax", "argmax"], ["quant", "argmax", "quant"]]
    # entries differ but every step agrees: no per-sample generators needed
    assert U.sampling_modes(["argmax", "argmax"], [5, None], 2, 3) == [["argmax", "argmax"]] * 3


@pytest.mark.parametrize("kw", [
    dict(mode=["multinomial", "argmax"]),                                  # wrong length
    dict(mode=["multinomial", "argmax", "sample"]),                       # unknown mode
    dict(mode=["multinomial", "argmax", 1]),
    dict(mode="argmax", sampling_quant_steps=[0, 1]),                     # wrong length
    dict(mode="argmax", sampling_quant_steps=[0, -1, 2]),                 # negative
    dict(mode="argmax", sampling_quant_steps=[0, 1.0, 2]),                # not an int
    dict(mode="argmax", sampling_quant_steps=[0, True, 2]),
    dict(mode=["multinomial", "argmax", "quant"], codebook=None),          # quant without a codebook
    dict(mode=["multinomial", "argmax", "argmax"], sampling_quant_steps=[None, None, 1], codebook=None),
    dict(mode=["multinomial", "argmax", "argmax"], generator=None),        # mixed modes on one stream
    dict(mode=["multinomial", "argmax", "argmax"], generator="one"),
    dict(mode=["multinomial", "argmax", "argmax"], exact=True),
])
def test_sampling_modes_rejects(kw):
    kw = dict(kw)
    args = dict(generator=["g0", "g1", "g2"], codebook=torch.zeros(1), exact=False, sampling_quant_steps=None)
    args.update(kw)
    with pytest.raises(ValueError):
        U.sampling_modes(args["mode"], args["sampling_quant_steps"], 3, 3, args["generator"], args["exact"], args["codebook"])


def test_check_mode_and_quant_steps():
    for md in ops.SAMPLING_MODES:
        assert ops.check_mode("mode", md) == md
    for bad in ("Multinomial", None, 0, ["argmax"]):
        with pytest.raises(ValueError):
            ops.check_mode("mode", bad)
    assert ops.check_quant_steps("q", None) is None and ops.check_quant_steps("q", 0) == 0 and ops.check_quant_steps("q", 6) == 6
    for bad in (-1, 1.5, "2", True, [1]):
        with pytest.raises(ValueError):
            ops.check_quant_steps("q", bad)
