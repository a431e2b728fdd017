"""Prompt-to-prompt injection without a GPU: the oracle against the reference fixture, argument validation in every entry point,
the per-step table, and the engine's admission grouping and step-table column."""
import collections

import pytest
import torch

from helpers import load_golden, oracle_cfg, t


def _fixture():
    cfg, sd, g = load_golden("paella_tiny.npz")
    _, _, z = load_golden("attention_source_tiny.npz")
    own = (t(g["byt5"]), t(g["clip"]), t(g["clip_image"]))
    same = (t(z["same_byt5"]), t(z["same_clip"]), t(z["same_clip_image"]))
    cases = {"prompt": (t(g["x"]), own, [None, 0], None),
             "attnw": (t(g["x"]), same, [None, 0], [None, t(g["attn_weights"])]),
             "x16": (t(z["x16"]), own, [None, 0], None),
             "self": (t(g["x"]), own, [0, 1], None)}
    return cfg, sd, g, z, cases


def test_oracle_matches_reference_fixture():
    # The reference runs in fp32; the oracle's fp32 forward agrees with it to ~1e-6 relative on logits of magnitude ~2
    # (test_oracle_golden), so 2e-5 absolute is a bound with room; the observed difference is ~2e-6.
    from oracle import attention_source as osrc
    cfg, sd, g, z, cases = _fixture()
    for name, (x, cond, src, w) in cases.items():
        got = osrc.paella_forward_injected(sd, oracle_cfg(cfg), x, t(g["r"]), *cond, src=src, attn_weights=w)
        want = t(z[f"logits_{name}"])
        assert got.shape == want.shape
        err = float((got - want).abs().max())
        assert err < 2e-5, (name, err)


def test_fixture_invariants():
    _, _, g, z, _ = _fixture()
    # a sample replaying itself is the plain forward; the source row of an edited batch is untouched; the edit is not
    assert torch.equal(t(z["logits_self"]), t(z["logits_plain"]))
    assert torch.equal(t(z["logits_prompt"])[0], t(z["logits_plain"])[0])
    assert float((t(z["logits_prompt"])[1] - t(z["logits_plain"])[1]).abs().max()) > 1e-2


# ------------------------------------------------------------------ validation: ValueError before any work
class _NoModel:
    """A stand-in model that fails on any use: the check must come first."""

    num_labels = 64

    def _device(self):
        return torch.device("cpu")

    def __getattr__(self, name):
        if name == "conditioning_seq_len":
            return lambda inputs: inputs["byt5"].shape[1]
        raise AssertionError(f"model.{name} used before the attention_source check")


def _inputs(B=2, L=3):
    return {"byt5": torch.randn(B, L, 8)}


_REGION = [(_inputs(1), torch.ones(4, 4, dtype=torch.bool))]
BAD = {
    "not-a-list": ({1: (0, 1)}, None, False),
    "length": ([None], None, False),
    "bool-source": ([None, (True, 1)], None, False),
    "bool-steps": ([None, (0, False)], None, False),
    "float": ([None, (0.0, 1)], None, False),
    "triple": ([None, (0, 1, 2)], None, False),
    "out-of-range": ([None, (2, 1)], None, False),
    "negative": ([None, (-1, 1)], None, False),
    "self": ([None, (1, 1)], None, False),
    "chain": ([(1, 1), (0, 1)], None, False),
    "k-too-large": ([None, (0, 3)], None, False),
    "k-negative": ([None, (0, -1)], None, False),
    "regions-on-edit": ([None, (0, 1)], [None, _REGION], False),
    "regions-on-source": ([None, (0, 1)], [_REGION, None], False),
    "exact": ([None, (0, 1)], None, True),
}


@pytest.mark.parametrize("case", sorted(BAD))
@pytest.mark.parametrize("entry", ["sample", "sample_distributed", "sample_notebook"])
def test_sampling_validation_before_any_work(entry, case):
    from paella_b200 import utils as U
    src, regions, exact = BAD[case]
    gens = [torch.Generator().manual_seed(5 + i) for i in range(2)]
    states = [g.get_state() for g in gens]
    with pytest.raises(ValueError, match="attention_source|exact"):
        if entry == "sample":
            U.sample(_NoModel(), _inputs(), (2, 4, 4), _inputs(), steps=2, generator=gens, prompt_regions=regions,
                     exact=exact, attention_source=src)
        elif entry == "sample_distributed":
            U.sample_distributed(_NoModel(), _inputs(), _inputs(), (2, 4, 4), steps=2, generator=gens, prompt_regions=regions,
                                 exact=exact, attention_source=src)
        else:
            U.sample_notebook(_NoModel(), _inputs(), (2, 4, 4), steps=2, generator=gens, prompt_regions=regions, exact=exact,
                              attention_source=src)
    assert all(torch.equal(g.get_state(), s) for g, s in zip(gens, states))


@pytest.mark.parametrize("src,regions", [({1: 0}, None), ([None], None), ([None, True], None), ([None, (0, 1)], None),
                                         ([None, 2], None), ([None, 1], None), ([1, 0], None), ([None, 0], [None, _REGION])],
                         ids=["not-a-list", "length", "bool", "pair", "out-of-range", "self", "chain", "regions"])
def test_forward_validation_before_any_work(src, regions):
    from paella_b200.modules import Paella
    cfg, _, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg)
    with pytest.raises(ValueError, match="attention_source"):
        Paella.forward(m, torch.zeros(2, 4, 4, dtype=torch.long), torch.zeros(2), torch.zeros(2, 3, cfg["byt5_embd"]), prompt_regions=regions,
                       attention_source=src)


# ------------------------------------------------------------------ the per-step table
def test_attention_source_table():
    from paella_b200 import ops
    assert ops.attention_source_table(None, 3, 4) is None
    assert ops.attention_source_table([None, None, None], 3, 4) is None
    tab = ops.attention_source_table([None, (0, 2), (0, 4)], 3, 4)
    assert tab.dtype == torch.int32 and tab.tolist() == [[-1, 0, 0], [-1, 0, 0], [-1, -1, 0], [-1, -1, 0]]
    # k = 0 everywhere: a table with no injected entry, so every step launches as without injection
    tab = ops.attention_source_table([(1, 0), None], 2, 3)
    assert tab.tolist() == [[-1, -1]] * 3
    # two edits of one source; a tuple or list pair
    assert ops.attention_source_table(((2, 1), [2, 3], None), 3, 3).tolist() == [[2, 2, -1], [-1, 2, -1], [-1, 2, -1]]
    # forward: ints, injected in the one forward
    assert ops.attention_source_table([None, 0], 2, 1, forward=True).tolist() == [[-1, 0]]
    # a sample without regions next to a regional one may be an edit
    regions = (torch.ones(3, 4, 4, dtype=torch.uint8), [[], [], [{"byt5": torch.zeros(1, 2, 8)}]])
    assert ops.attention_source_table([None, (0, 1), None], 3, 2, regions).tolist() == [[-1, 0, -1], [-1, -1, -1]]


# ------------------------------------------------------------------ engine
def _request(steps=4, guided=True, cond_len=5, renoise=None, cond_steps=None, source=None):
    from paella_b200.engine import Request
    q = Request(steps, steps - 1 if renoise is None else renoise, steps if cond_steps is None else cond_steps, guided,
                torch.zeros(steps, 3), torch.zeros(steps + 1), maps_len=cond_len, attention_source=source)
    if source is not None:
        source[0].edits.append(q)
    return q


def test_engine_admission_groups_a_source_with_its_edits():
    from paella_b200.engine import admit_from_queue
    a = _request()
    b = _request()
    e1 = _request(source=(b, 2))
    c = _request()
    e2 = _request(source=(b, 4))
    queue = collections.deque([a, b, e1, c, e2])
    # 2 free slots: a, then b needs 3 -> waits, and c behind it waits too (FIFO)
    assert admit_from_queue(queue, 2) == [a]
    assert list(queue) == [b, e1, c, e2]
    assert admit_from_queue(queue, 2) == []
    # 4 free slots: b with both edits, then c
    assert admit_from_queue(queue, 4) == [b, e1, e2, c]
    assert not queue


def test_engine_inj_src_column_under_guided_first_order():
    from paella_b200.engine import build_step_plan, step_host_table
    src = _request(guided=False)
    edit = _request(guided=True, source=(src, 2))
    other = _request(guided=True)
    for q, slot in ((src, 0), (edit, 1), (other, 2)):
        q.slot, q.uncond_slot = slot, 8 + slot
    plan = build_step_plan([src, edit, other])
    # guided first: edit (row 0), other (row 1), then the source (row 2)
    assert plan.order == [edit, other, src]
    assert plan.injects and plan.inj_src.dtype == torch.int32 and plan.inj_src.tolist() == [2, -1, -1]
    host, lay = step_host_table(plan, [0, 0] * 3, [0, 0] * 3)
    dt, o, n = lay["inj_src"]
    i32 = host[lay["i32"][1]:lay["i32"][1] + lay["i32"][2]].view(torch.int32)
    assert dt == "i32" and i32[o:o + n].tolist() == [2, -1, -1]
    d2, o2, n2 = lay["kv_slot"]
    assert i32[o2:o2 + n2].tolist() == plan.kv_slot.tolist()
    # past the window: no column, the layout of a step without edits
    for q in (src, edit, other):
        q.k = 2
    plan = build_step_plan([src, edit, other])
    assert not plan.injects
    _, lay = step_host_table(plan, [0, 0] * 3, [0, 0] * 3)
    assert [k for k, v in lay.items() if v[0] == "i32"] == ["row_slot", "kv_slot", "modes"]


class _EngineStub:
    """The attributes SamplingEngine._check_attention_source reads."""

    def __init__(self, queue, max_batch=4):
        from paella_b200.engine import SamplingEngine
        self._queue = collections.deque(queue)
        self.max_batch = max_batch
        self.model = _NoModel()
        self.check = lambda *a: SamplingEngine._check_attention_source(self, *a)


@pytest.mark.parametrize("case", ["not-a-pair", "not-a-request", "bool-k", "not-queued", "chain", "regions-on-edit",
                                  "regions-on-source", "cond-len", "steps", "renoise", "cond-steps", "k-too-large",
                                  "max-batch"])
def test_engine_submit_rules(case):
    src = _request(steps=4)
    edit_of_src = _request(steps=4, source=(src, 1))
    queue = [src, edit_of_src]
    args = dict(attention_source=(src, 2), byt5_len=5, steps=4, renoise=3, cond_steps=4, regions=None)
    if case == "not-a-pair":
        args["attention_source"] = src
    elif case == "not-a-request":
        args["attention_source"] = (0, 2)
    elif case == "bool-k":
        args["attention_source"] = (src, True)
    elif case == "not-queued":
        queue = []
    elif case == "chain":
        args["attention_source"] = (edit_of_src, 2)
    elif case == "regions-on-edit":
        args["regions"] = _REGION
    elif case == "regions-on-source":
        src.regional = True
    elif case == "cond-len":
        args["byt5_len"] = 6
    elif case == "steps":
        args["steps"] = 5
    elif case == "renoise":
        args["renoise"] = 2
    elif case == "cond-steps":
        args["cond_steps"] = 3
    elif case == "k-too-large":
        args["attention_source"] = (src, 5)
    eng = _EngineStub(queue, max_batch=2 if case == "max-batch" else 4)
    inputs = {"byt5": torch.zeros(1, args["byt5_len"], 8)}
    with pytest.raises(ValueError, match="attention_source"):
        eng.check(args["attention_source"], inputs, args["steps"], args["renoise"], args["cond_steps"], args["regions"])
    # the same request passes with the defaults
    if case not in ("not-queued", "max-batch", "regions-on-source"):
        eng.check((src, 2), {"byt5": torch.zeros(1, 5, 8)}, 4, 3, 4, None)
