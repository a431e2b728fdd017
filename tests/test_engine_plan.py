"""SamplingEngine's per-step table builder, without a device: for requests at different step indices, the batch is ordered
guided first, and each row carries its own request's schedule row (utils.sampling_schedule at batch 1), renoise target,
guided flag and slots."""
import random

import torch

from paella_b200 import utils as U
from paella_b200.engine import Request, build_step_plan


def _request(rng, slot, shared_uncond):
    steps = rng.choice([1, 3, 5, 8, 12])
    cfg = rng.choice([None, (8.0, 8.0), (9.0, 2.5)])
    temperature = (rng.uniform(0.2, 1.5), rng.uniform(0.2, 1.5))
    t_start, t_end = rng.uniform(0.6, 1.0), rng.uniform(0.0, 0.3)
    renoise = rng.choice([None, 0, steps // 2, steps + 1])
    renoise = steps - 1 if renoise is None else renoise
    cond_steps = rng.choice([steps, max(1, steps // 2), 0])
    cfgs = U._cfg_schedule(cfg, 1, steps)
    params, r = U.sampling_schedule(1, steps, temperature, cfgs, t_start, t_end, always=True)
    q = Request(steps, renoise, cond_steps, cfg is not None, params[:, 0], r[:, 0])
    q.slot = slot
    q.uncond_slot = 100 if shared_uncond else 50 + slot
    q.k = rng.randrange(steps)
    q.spec = dict(steps=steps, cfgs=cfgs, temperature=temperature, t_start=t_start, t_end=t_end)
    return q


def test_step_plan_rows_follow_each_request_schedule():
    rng = random.Random(0)
    for trial in range(200):
        n = rng.randint(1, 12)
        slots = rng.sample(range(40), n)
        active = [_request(rng, s, rng.random() < 0.5) for s in slots]
        plan = build_step_plan(active)
        assert sorted(id(q) for q in plan.order) == sorted(id(q) for q in active)
        guided = [q.guided and q.k < q.cond_steps for q in plan.order]
        assert plan.n_pairs == sum(guided)
        assert guided == sorted(guided, reverse=True), "guided rows must come first"
        # each group keeps admission order
        pos = {id(q): i for i, q in enumerate(active)}
        for grp in (plan.order[:plan.n_pairs], plan.order[plan.n_pairs:]):
            assert [pos[id(q)] for q in grp] == sorted(pos[id(q)] for q in grp)
        for i, q in enumerate(plan.order):
            s = q.spec
            params, r = U.sampling_schedule(1, s["steps"], s["temperature"], s["cfgs"], s["t_start"], s["t_end"], always=True)
            assert torch.equal(plan.params[i], params[q.k, 0])
            assert torch.equal(plan.r[i], r[q.k, 0])
            if q.k < q.renoise_steps:
                assert plan.renoise[i] and torch.equal(plan.t_next[i], r[q.k + 1, 0])
            else:
                assert not plan.renoise[i] and float(plan.t_next[i]) < 0
            if s["cfgs"] is not None:        # the fp32 constants of the scalar path
                c = s["cfgs"][q.k]
                assert float(plan.params[i, 0]) == float(torch.tensor(c, dtype=torch.float64).float())
                assert float(plan.params[i, 1]) == float(torch.tensor(1.0 - c, dtype=torch.float64).float())
            t = torch.linspace(s["temperature"][0], s["temperature"][1], s["steps"])[q.k]
            assert float(plan.params[i, 2]) == float(torch.ones(()) / t)
        assert plan.row_slot.dtype == torch.int32 and plan.row_slot.tolist() == [q.slot for q in plan.order]
        assert plan.kv_slot.tolist() == [q.slot for q in plan.order] + [q.uncond_slot for q in plan.order[:plan.n_pairs]]


def test_sampling_schedule_always_matches_the_per_sample_table():
    """``always=True`` on scalar arguments gives what a per-sample tensor of the same values gives."""
    cfgs = U._cfg_schedule((7.0, 3.0), 1, 6)
    a = U.sampling_schedule(1, 6, (0.9, 0.4), cfgs, 0.95, 0.05, always=True)
    b = U.sampling_schedule(1, 6, torch.tensor([[0.9, 0.4]]), cfgs, torch.tensor([0.95]), torch.tensor([0.05]))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert U.sampling_schedule(1, 6, (0.9, 0.4), cfgs, 0.95, 0.05) is None
