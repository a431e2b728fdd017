"""Guidance prompts without a GPU: argument validation, the mix coefficients and tables, the engine's step plan, and the oracle's
fp64 mix against a plain torch float64 formulation."""
import math
import random

import pytest
import torch

from helpers import load_golden, oracle_cfg, t


def _inputs(L=3):
    return {"byt5": torch.randn(1, L, 8)}


# ------------------------------------------------------------------ validation
def test_guidance_table_layout():
    from paella_b200 import ops
    p1, p2, p3 = _inputs(), _inputs(5), _inputs(2)
    terms = ops.guidance_table([[(p1, 0.5), (p2, -1)], None, [(p3, 2.0)]], 3)
    assert terms == [[(p1, 0.5), (p2, -1.0)], [], [(p3, 2.0)]]
    assert all(isinstance(w, float) for own in terms for _, w in own)
    assert ops.guidance_table(None, 2) is None
    assert ops.guidance_table([None, []], 2) is None
    assert len(ops.guidance_table([[(p1, 1.0)] * ops.MAX_GUIDANCE_PROMPTS], 1)[0]) == 7


@pytest.mark.parametrize("bad", [
    "x", [None], [[(None, None)]] * 2, [[(_inputs(),)], None], [(_inputs(), 1.0), None],
    [[(_inputs(), 1.0)] * 8, None],                                    # more than 7 terms
    [[(_inputs(), float("nan"))], None], [[(_inputs(), float("inf"))], None], [[(_inputs(), -float("inf"))], None],
    [[(_inputs(), "1")], None], [[(_inputs(), True)], None], [[(_inputs(), torch.tensor(1.0))], None],
    [[({"byt5": torch.randn(2, 3, 8)}, 1.0)], None],                   # batch-2 inputs
    [[({"byt5": torch.randn(1, 3, 8), "clip": torch.randn(2, 8)}, 1.0)], None],
    [[({"clip": torch.randn(1, 8)}, 1.0)], None],
])
def test_guidance_table_rejects(bad):
    from paella_b200 import ops
    with pytest.raises(ValueError):
        ops.guidance_table(bad, 2)


# ------------------------------------------------------------------ coefficients
def test_coefficients_without_terms_are_the_cfg_constants():
    from paella_b200 import ops
    rng = random.Random(0)
    cfgs = [8.0, 1.0, 0.5, 3.0000001, -2.5, 1e-7] + [rng.uniform(-20, 20) for _ in range(200)]
    want = ops.sampling_params([[c] for c in cfgs], [[1.0]] * len(cfgs))[:, 0, :2]
    got = torch.tensor([ops.guidance_coefficients(c, []) for c in cfgs], dtype=torch.float32)
    assert torch.equal(got.view(torch.int32), want.contiguous().view(torch.int32))
    # torch.linspace schedules, as sample_distributed builds them
    for a, b in ((8.0, 2.0), (7.5, 7.5), (1.3, 11.1)):
        sched = torch.linspace(a, b, 12).tolist()
        want = ops.sampling_params([sched], [[1.0] * 12])[0, :, :2]
        got = torch.tensor([ops.guidance_coefficients(c, []) for c in sched], dtype=torch.float32)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32))


def test_coefficients_with_terms_are_the_double_formula_rounded():
    import numpy as np
    from paella_b200 import ops
    rng = random.Random(1)
    for _ in range(300):
        c = rng.uniform(-12, 12)
        ws = [rng.uniform(-3, 3) for _ in range(rng.randint(1, 7))]
        got = ops.guidance_coefficients(c, ws)
        s = 0.0
        for w in ws:
            s += w
        want = [np.float32(c), np.float32(1.0 - c * (1.0 + s))] + [np.float32(c * w) for w in ws]
        assert [np.float32(v) for v in got] == want
        assert all(isinstance(v, float) and math.isfinite(v) for v in got)
        assert abs(sum(got) - 1.0) < 1e-5 * (1 + abs(c) * (1 + sum(abs(w) for w in ws)))


def test_mix_table_layout():
    from paella_b200 import ops
    rows, coef = ops.guidance_mix_table([[0.5, -1.0], [2.0]], [1, 3], [5, 7], [[8, 9], [10]], [[4.0, 6.0], [3.0, 2.0], [1.5, 1.0]])
    assert rows.dtype == torch.int32 and rows.tolist() == [[1, 5, 8, 9], [3, 7, 10, -1]]
    assert coef.dtype == torch.float32 and coef.shape == (3, 2, 4)
    for i, cs in enumerate([[4.0, 6.0], [3.0, 2.0], [1.5, 1.0]]):
        assert coef[i, 0].tolist() == ops.guidance_coefficients(cs[0], [0.5, -1.0])
        assert coef[i, 1, :3].tolist() == ops.guidance_coefficients(cs[1], [2.0]) and coef[i, 1, 3] == 0


# ------------------------------------------------------------------ engine step plan
def _request(rng, slot, steps, terms=0, cfg=(8.0, 3.0), cond_steps=None):
    from paella_b200 import ops
    from paella_b200 import utils as U
    from paella_b200.engine import Request
    cond_steps = steps if cond_steps is None else cond_steps
    cfgs = U._cfg_schedule(cfg, 1, steps)
    params, r = U.sampling_schedule(1, steps, (1.0, 0.3), cfgs, 1.0, 0.0, always=True)
    tl = [({"byt5": torch.zeros(1, 2, 4)}, rng.uniform(-2, 2)) for _ in range(terms)] or None
    mix = None
    if tl:
        mix = torch.tensor([ops.guidance_coefficients(cfgs[i], [w for _, w in tl]) for i in range(min(steps, cond_steps))],
                           dtype=torch.float32)
        params[:min(steps, cond_steps), 0, :2] = torch.tensor([1.0, 0.0])
    q = Request(steps, steps - 1, cond_steps, cfgs is not None, params[:, 0], r[:, 0], terms=tl, mix_coef=mix)
    q.slot, q.uncond_slot = slot, 100 + slot
    q.term_slot = [200 + 10 * slot + j for j in range(terms)]
    return q


def test_engine_step_plan_layout():
    from paella_b200.engine import build_step_plan, step_host_table
    rng = random.Random(3)
    qs = [_request(rng, 0, 4, terms=2), _request(rng, 1, 4), _request(rng, 2, 4, terms=1, cond_steps=2),
          _request(rng, 3, 4, cfg=None), _request(rng, 4, 4, terms=3)]
    for step in range(4):
        for q in qs:
            q.k = step
        plan = build_step_plan(qs)
        order = plan.order
        Bc, n_pairs = len(order), plan.n_pairs
        guided = [q for q in order[:n_pairs]]
        comp = [i for i, q in enumerate(guided) if q.n_terms]
        assert plan.composed == comp
        assert order[n_pairs:] == [q for q in qs if not (q.guided and q.k < q.cond_steps)]
        # tail: the unconditional rows of the guided, then each composed row's terms in order
        want_tail = list(range(n_pairs)) + [i for i in comp for _ in range(order[i].n_terms)]
        assert plan.tail.tolist() == want_tail
        want_kv = [q.slot for q in order] + [q.uncond_slot for q in guided] + [s for i in comp for s in order[i].term_slot]
        assert plan.kv_slot.tolist() == want_kv
        t0 = Bc + n_pairs
        for y, i in enumerate(comp):
            q = order[i]
            assert plan.mix_rows[y, :2 + q.n_terms].tolist() == [i, Bc + i] + list(range(t0, t0 + q.n_terms))
            assert bool((plan.mix_rows[y, 2 + q.n_terms:] == -1).all())
            assert torch.equal(plan.mix_coef[y, :2 + q.n_terms], q.mix_coef[q.k])
            assert plan.params[i, 0] == 1.0 and plan.params[i, 1] == 0.0
            t0 += q.n_terms
        host, lay = step_host_table(plan, [0, 0] * Bc, [0, 0] * Bc)
        assert ("tail" in lay) == bool(comp) and ("mix_rows" in lay) == bool(comp) and ("mix_coef" in lay) == bool(comp)
        if comp:
            i32 = host[lay["i32"][1]:lay["i32"][1] + lay["i32"][2]].view(torch.int32)
            f32 = host[lay["f32"][1]:lay["f32"][1] + lay["f32"][2]].view(torch.float32)
            _, o, n = lay["tail"]
            assert i32[o:o + n].tolist() == want_tail
            _, o, n = lay["mix_rows"]
            assert torch.equal(i32[o:o + n], plan.mix_rows.view(-1))
            _, o, n = lay["mix_coef"]
            assert torch.equal(f32[o:o + n], plan.mix_coef.view(-1))
    assert qs[2].k == 3 and 2 not in [q.slot for q in build_step_plan(qs).order[:build_step_plan(qs).n_pairs]]


def test_engine_plan_without_terms_is_unchanged():
    """Requests without terms: the step's host table has exactly the parent's parts and values."""
    from paella_b200.engine import build_step_plan, step_host_table
    rng = random.Random(4)
    qs = [_request(rng, 0, 3), _request(rng, 1, 3, cfg=None), _request(rng, 2, 3)]
    plan = build_step_plan(qs)
    assert plan.composed == [] and plan.kv_slot.tolist() == [0, 2, 1, 100, 102]
    host, lay = step_host_table(plan, [0, 0] * 3, [0, 0] * 3)
    assert set(lay) == {"r", "params", "t_next", "row_slot", "kv_slot", "modes", "f32", "i32", "u8"}
    assert lay["f32"][2] == (3 * 5 + 1) // 2 and lay["i32"][2] == (3 + 5 + 1) // 2 and lay["u8"][2] == 0
    assert host.numel() == 4 * 3 + lay["f32"][2] + lay["i32"][2]


def test_engine_slots_are_disjoint():
    """_term_slot lies after the regional slots and never collides (the engine arithmetic, without a model)."""
    from paella_b200.engine import SamplingEngine
    e = SamplingEngine.__new__(SamplingEngine)
    e.max_batch, e.max_regions, e.max_terms = 5, 2, 3
    seen = {2 * e.max_batch}
    seen |= set(range(2 * e.max_batch))
    for s in range(e.max_batch):
        for k in range(e.max_regions):
            seen.add(e._region_slot(s, k))
    n = len(seen)
    terms = {e._term_slot(s, j) for s in range(e.max_batch) for j in range(e.max_terms)}
    assert not (terms & seen) and len(terms) == e.max_batch * e.max_terms
    assert max(terms) == 2 * e.max_batch + 1 + (e.max_regions + e.max_terms) * e.max_batch - 1 and n == 2 * 5 + 1 + 2 * 5


# ------------------------------------------------------------------ oracle
def test_oracle_mix_against_plain_float64():
    from oracle import guidance as og
    g = torch.Generator().manual_seed(0)
    c, u = torch.randn(2, 16, 4, 4, generator=g), torch.randn(2, 16, 4, 4, generator=g)
    ts = [torch.randn(2, 16, 4, 4, generator=g) for _ in range(3)]
    ws = [0.5, -1.25, 2.0]
    got = og.mix(c, u, ts, 7.5, ws)
    a = og.coefficients(7.5, ws)
    want = a[0] * c.double() + a[1] * u.double() + sum(aj * tj.double() for aj, tj in zip(a[2:], ts))
    assert got.dtype == torch.float64
    assert float((got - want).abs().max()) < 1e-12
    assert abs(sum(a) - 1.0) < 1e-12
    assert torch.equal(og.mix(c, u, [], 3.0, []), u.double() + 3.0 * (c.double() - u.double()))


def test_oracle_guided_logits_on_the_tiny_model():
    """guided_logits is the mix of three ordinary oracle forwards, and a weight-0 term leaves plain CFG."""
    from oracle import guidance as og
    from oracle import paella_oracle as po
    cfg, sd, g = load_golden("paella_tiny.npz")
    oc = oracle_cfg(cfg)
    x, r = t(g["x"]), t(g["r"])
    cond = dict(byt5=t(g["byt5"]), clip=t(g["clip"]))
    uncond = {k: torch.zeros_like(v) for k, v in cond.items()}
    term = dict(byt5=t(g["byt5"][1:2]), clip=t(g["clip"][:1]))
    got = og.guided_logits(sd, oc, x, r, cond, uncond, [term], 4.0, [0.5])
    lc = po.paella_forward(sd, oc, x, r, cond["byt5"], cond["clip"]).double()
    lu = po.paella_forward(sd, oc, x, r, uncond["byt5"], uncond["clip"]).double()
    lt = po.paella_forward(sd, oc, x, r, term["byt5"].expand(2, -1, -1), term["clip"].expand(2, -1)).double()
    assert float((got - (lu + 4.0 * ((lc - lu) + 0.5 * (lt - lu)))).abs().max()) < 1e-9
    zero = og.guided_logits(sd, oc, x, r, cond, uncond, [term], 4.0, [0.0])
    assert float((zero - (lu + 4.0 * (lc - lu))).abs().max()) < 1e-9
