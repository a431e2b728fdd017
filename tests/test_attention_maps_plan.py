"""Attention maps without a GPU: the oracle against the reference fixture, argument validation in every entry point, and the
host tables (engine map rows, accumulator layout)."""
import pytest
import torch

from helpers import load_golden, oracle_cfg, t


def _fixture():
    cfg, sd, g = load_golden("paella_tiny.npz")
    _, _, z = load_golden("attention_maps_tiny.npz")
    ci = t(g["clip_image"])
    cases = {"plain": (t(g["x"]), dict(clip_image=ci)),
             "attnw": (t(g["x"]), dict(clip_image=ci, attn_weights=t(g["attn_weights"]))),
             "x16": (t(z["x16"]), dict(clip_image=ci)),
             "img2": (t(g["x"]), dict(clip_image=[ci, t(z["clip_image2"])]))}
    return cfg, sd, g, z, cases


def test_oracle_matches_reference_fixture():
    # The reference's matrices are fp32 softmax outputs of its fp32 forward; the oracle's fp32 forward agrees with it to ~1e-5
    # relative on the logits (test_oracle_golden), and a probability p moves by about p * |d score| under such a perturbation of
    # q and k, so 1e-6 absolute on maps of at most 1 is a bound with room; the observed difference is ~1e-8.
    from oracle import attention_maps as om
    cfg, sd, g, z, cases = _fixture()
    for name, (x, kw) in cases.items():
        _, maps = om.paella_maps(sd, oracle_cfg(cfg), x, t(g["r"]), t(g["byt5"]), t(g["clip"]), **kw)
        want = t(z[f"maps_{name}"]).double()
        assert maps.dtype == torch.float64 and maps.shape == want.shape
        err = float((maps - want).abs().max())
        assert err < 1e-6, (name, err)
    # the weights matter
    assert float((t(z["maps_attnw"]) - t(z["maps_plain"])).abs().max()) > 1e-3


def test_oracle_invariants():
    from oracle import attention_maps as om
    cfg, sd, g, z, cases = _fixture()
    x, kw = cases["x16"]
    _, maps = om.paella_maps(sd, oracle_cfg(cfg), x, t(g["r"]), t(g["byt5"]), t(g["clip"]), **kw)
    assert bool((maps >= 0).all())
    assert float(maps.sum(1).max()) <= 1.0 + 1e-12        # the self keys take the rest of each softmax
    # nearest-neighbour upsampling: a 4 x 4 token footprint of the finest AttnBlock level holds one value
    assert torch.equal(maps[..., 0::4, 0::4], maps[..., 3::4, 3::4])


# ------------------------------------------------------------------ validation: ValueError before any work
class _NoModel:
    """A stand-in model that fails on any use: the check must come first."""

    def __getattr__(self, name):
        raise AssertionError(f"model.{name} used before the attention_maps check")


def _inputs(L=3):
    return {"byt5": torch.randn(1, L, 8)}


_REGIONS = [[(_inputs(), torch.ones(4, 4, dtype=torch.bool))]]


@pytest.mark.parametrize("flag,regions", [("yes", None), (1, None), (None, None), (torch.tensor(True), None), (True, _REGIONS)],
                         ids=["str", "int", "none", "tensor", "with-regions"])
@pytest.mark.parametrize("entry", ["sample", "sample_distributed", "sample_notebook", "forward", "submit"])
def test_validation_before_any_work(entry, flag, regions):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    from paella_b200.modules import Paella
    g = torch.Generator().manual_seed(5)
    state = g.get_state()
    m = _NoModel()
    with pytest.raises(ValueError, match="attention_maps"):
        if entry == "sample":
            U.sample(m, _inputs(), (1, 4, 4), _inputs(), generator=[g], prompt_regions=regions, attention_maps=flag)
        elif entry == "sample_distributed":
            U.sample_distributed(m, _inputs(), _inputs(), (1, 4, 4), generator=[g], prompt_regions=regions, attention_maps=flag)
        elif entry == "sample_notebook":
            U.sample_notebook(m, _inputs(), (1, 4, 4), generator=[g], prompt_regions=regions, attention_maps=flag)
        elif entry == "forward":
            Paella.forward(object.__new__(Paella), torch.zeros(1, 4, 4, dtype=torch.long), torch.zeros(1), torch.zeros(1, 3, 8),
                           prompt_regions=regions, attention_maps=flag)
        else:
            SamplingEngine.submit(object.__new__(SamplingEngine), _inputs(), generator=g,
                                  prompt_regions=regions[0] if regions else None, attention_maps=flag)
    assert torch.equal(g.get_state(), state)


def test_flag_values():
    from paella_b200 import ops
    assert ops.check_attention_maps(False) is False and ops.check_attention_maps(True) is True
    assert ops.check_attention_maps(False, _REGIONS) is False


# ------------------------------------------------------------------ host tables
def _request(slot, steps, maps, guided=True, cond_len=5):
    from paella_b200.engine import Request
    q = Request(steps, steps - 1, steps, guided, torch.zeros(steps, 3), torch.zeros(steps + 1), attention_maps=maps,
                maps_len=cond_len)
    q.slot, q.uncond_slot = slot, 8 + slot
    return q


def test_engine_map_rows_in_the_step_table():
    from paella_b200.engine import build_step_plan, step_host_table
    qs = [_request(3, 4, True), _request(0, 6, False, guided=False), _request(5, 2, True, guided=False, cond_len=9),
          _request(1, 3, False)]
    plan = build_step_plan(qs)
    # guided rows first: slots 3, 1, then 0, 5
    assert [q.slot for q in plan.order] == [3, 1, 0, 5]
    assert plan.maps and plan.map_row.dtype == torch.int32 and plan.map_row.tolist() == [3, -1, -1, 5]
    Bc = len(qs)
    host, lay = step_host_table(plan, [0, 0] * Bc, [0, 0] * Bc)
    dt, o, n = lay["map_row"]
    assert dt == "i32" and n == Bc
    i32 = host[lay["i32"][1]:lay["i32"][1] + lay["i32"][2]].view(torch.int32)
    assert i32[o:o + n].tolist() == [3, -1, -1, 5]
    # the kv_slot part is unchanged by the map rows
    d2, o2, n2 = lay["kv_slot"]
    assert i32[o2:o2 + n2].tolist() == plan.kv_slot.tolist()


def test_engine_step_without_maps_has_the_parent_layout():
    from paella_b200.engine import build_step_plan, step_host_table
    qs = [_request(2, 4, False), _request(0, 3, False, guided=False)]
    plan = build_step_plan(qs)
    assert not plan.maps
    host, lay = step_host_table(plan, [0, 0] * 2, [0, 0] * 2)
    assert "map_row" not in lay
    assert [k for k, v in lay.items() if v[0] == "i32"] == ["row_slot", "kv_slot", "modes"]


def test_accumulator_layout():
    from paella_b200.modules import Paella
    cfg, _, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg)
    # patch 2, three levels: block grids 4x4, 2x2, 1x1 at 8x8 tokens; level 0 first
    assert m.map_positions((8, 8)) == 16 + 4 + 1
    assert m.map_positions((16, 32)) == 8 * 16 + 4 * 8 + 2 * 4
