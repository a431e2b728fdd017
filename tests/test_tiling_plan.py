"""Seamless tiling without a device: the wrap-around oracle against the reference's circular-padding run
(tests/golden/tiling_tiny.npz), argument validation and the host table (ops.tiling_table), validation at every entry point
before any work, and SamplingEngine's per-step table layout."""
import random

import pytest
import torch

from helpers import load_golden, oracle_cfg, t
from oracle import paella_oracle as po
from oracle import tiling as ot
from paella_b200 import ops
from paella_b200 import utils as U
from paella_b200.engine import Request, build_step_plan, step_host_table


# ------------------------------------------------------------------ the oracle against the reference
@pytest.mark.parametrize("tiling", ["xy", "x", "y"])
def test_denoiser_oracle_matches_reference_circular(tiling):
    cfg, sd, g = load_golden("paella_tiny.npz")
    _, _, z = load_golden("tiling_tiny.npz")
    got = ot.paella_forward(sd, oracle_cfg(cfg), t(g["x"]), t(g["r"]), t(g["byt5"]), t(g["clip"]), t(g["clip_image"]),
                            wrap=ot.WRAPS[tiling])
    want = t(z["logits_" + tiling])
    assert float((got - want).abs().max()) < 2e-4            # test_oracle_golden.py's logits bound
    assert float((t(g["logits"]) - want).abs().max()) > 0.1  # and the fixture is not the untiled forward


def test_untiled_oracle_is_the_paella_oracle():
    cfg, sd, g = load_golden("paella_tiny.npz")
    args = (sd, oracle_cfg(cfg), t(g["x"]), t(g["r"]), t(g["byt5"]), t(g["clip"]), t(g["clip_image"]))
    assert torch.equal(ot.paella_forward(*args), po.paella_forward(*args))


@pytest.mark.parametrize("tiling", ["xy", "x"])
def test_decoder_oracle_matches_reference_circular(tiling):
    vcfg, vsd, vg = load_golden("vqgan_tiny.npz")
    _, _, z = load_golden("tiling_tiny.npz")
    got = ot.decode_indices(vsd, t(z["idx"]), vcfg["bottleneck_blocks"], wrap=ot.WRAPS[tiling])
    want = t(z["dec_" + tiling])
    assert float((got - want).abs().max()) < 1e-4
    assert float((t(vg["dec_rand"]) - want).abs().max()) > 0.05


@pytest.mark.parametrize("hw", [(1, 1), (2, 3), (5, 4)])
def test_wrapped_conv_transpose_is_a_mod_n_sum(hw):
    """The kernel's definition (input indices mod n) against a direct fp64 sum, and the pad / conv / crop restatement."""
    h, w = hw
    g = torch.Generator().manual_seed(h * 7 + w)
    x = torch.randn(2, h, w, 3, dtype=torch.float64, generator=g)
    W = torch.randn(3, 5, 4, 4, dtype=torch.float64, generator=g)
    b = torch.randn(5, dtype=torch.float64, generator=g)
    want = torch.zeros(2, 2 * h, 2 * w, 5, dtype=torch.float64) + b
    for oy in range(2 * h):
        for ox in range(2 * w):
            for ky in range(4):
                for kx in range(4):
                    if (oy + 1 - ky) % 2 or (ox + 1 - kx) % 2:
                        continue
                    iy, ix = ((oy + 1 - ky) // 2) % h, ((ox + 1 - kx) // 2) % w
                    want[:, oy, ox] += x[:, iy, ix] @ W[:, :, ky, kx]
    got = ot.convT_k4s2p1_wrap(x, W, b, (True, True), mm=lambda a, m: a @ m.t())
    assert float((got - want).abs().max()) < 1e-12
    via_torch = ot.convT_circular_torch(x.permute(0, 3, 1, 2), W, b).permute(0, 2, 3, 1)
    assert float((via_torch - want).abs().max()) < 1e-12


def test_small_grid_depthwise_wraps_onto_itself():
    """On a 1x1 grid every tap of a wrapped k x k conv reads the one position; on a 2x2 grid a 5x5 kernel reads each position
    several times."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, 1, 1, 8, dtype=torch.float64, generator=g)
    w = torch.randn(8, 1, 3, 3, dtype=torch.float64, generator=g)
    b = torch.randn(8, dtype=torch.float64, generator=g)
    got = ot.dwconv_nhwc(x, w, b, wrap=(True, True))
    assert torch.allclose(got[0, 0, 0], b + x[0, 0, 0] * w[:, 0].sum((1, 2)))
    x2 = torch.randn(1, 2, 2, 8, dtype=torch.float64, generator=g)
    w5 = torch.randn(8, 1, 5, 5, dtype=torch.float64, generator=g)
    got = ot.dwconv_nhwc(x2, w5, b, wrap=(True, True))
    want = torch.zeros(1, 2, 2, 8, dtype=torch.float64) + b
    for y in range(2):
        for xx in range(2):
            for ky in range(5):
                for kx in range(5):
                    want[0, y, xx] += x2[0, (y + ky - 2) % 2, (xx + kx - 2) % 2] * w5[:, 0, ky, kx]
    assert float((got - want).abs().max()) < 1e-12


# ------------------------------------------------------------------ validation and the table
@pytest.mark.parametrize("tiling", ["xz", "XY", 1, True, ["x"], ["x", "q"], ("x", "y", "xy"), torch.tensor([1, 0]), [None, 3],
                                    [["x"], "y"]])
def test_bad_tiling_raises(tiling):
    with pytest.raises(ValueError):
        ops.tiling_table(tiling, 2)


def test_table_values():
    assert ops.tiling_table(None, 3) is None
    assert ops.tiling_table("none", 3) is None
    assert ops.tiling_table([None, "none"], 2) is None
    tab = ops.tiling_table("xy", 2)
    assert tab.dtype == torch.uint8 and tab.tolist() == [3, 3]
    assert ops.tiling_table(["none", "x", "y", "xy", None], 5).tolist() == [0, 1, 2, 3, 0]
    assert ops.tiling_table(("x",), 1).tolist() == [1]


class _NoDevice:
    """A stand-in model that fails on any device use: validation must come first."""
    num_labels = 64

    def _device(self):
        return torch.device("cpu")

    def __getattr__(self, name):
        raise AssertionError(f"model.{name} touched before validation")


@pytest.mark.parametrize("tiling", ["z", ["x"], torch.tensor([1, 1])])
def test_sampling_entry_points_validate_first(tiling):
    gens = [torch.Generator(), torch.Generator()]
    states = [g.get_state() for g in gens]
    for call in (lambda: U.sample(_NoDevice(), {}, (2, 4, 4), None, cfg=0, tiling=tiling, generator=gens),
                 lambda: U.sample_distributed(_NoDevice(), {}, None, (2, 4, 4), cfg=None, tiling=tiling, generator=gens),
                 lambda: U.sample_notebook(_NoDevice(), {"byt5": torch.zeros(2, 1, 4)}, (2, 4, 4), cfg=None, tiling=tiling,
                                           generator=gens)):
        with pytest.raises(ValueError, match="tiling"):
            call()
    assert all(torch.equal(a, g.get_state()) for a, g in zip(states, gens))


# ------------------------------------------------------------------ the engine's per-step table
def _request(rng, slot, steps, wrap, top_k=0):
    cfg = rng.choice([None, (8.0, 8.0)])
    cfgs = U._cfg_schedule(cfg, 1, steps)
    params, r = U.sampling_schedule(1, steps, (0.7, 0.3), cfgs, 1.0, 0.0, always=True)
    q = Request(steps, steps - 1, steps, cfg is not None, params[:, 0], r[:, 0], top_k=top_k, wrap=wrap)
    q.slot, q.uncond_slot = slot, 99
    return q


def test_step_table_carries_wrap_bytes_only_when_a_row_wraps():
    rng = random.Random(7)
    seen = set()
    for trial in range(40):
        reqs = [_request(rng, j, rng.choice([1, 2, 4]), rng.choice([0, 0, 0, 1, 2, 3]), rng.choice([0, 0, 5]))
                for j in range(rng.randint(1, 9))]
        active = list(reqs)
        while active:
            plan = build_step_plan(active)
            Bc = len(plan.order)
            wraps = any(q.wrap for q in plan.order)
            seen.add(wraps)
            assert plan.wraps == wraps
            host, lay = step_host_table(plan, [0, 0] * Bc, [0, 0] * Bc)
            untiled = lay["u8"][2] == 0
            if wraps:
                u8 = host[lay["u8"][1]:lay["u8"][1] + lay["u8"][2]].view(torch.uint8)
                dt, o, n = lay["wrap"]
                assert dt == "u8" and u8[o:o + n].tolist() == [q.wrap for q in plan.order]
                assert lay["u8"][2] == (Bc + 7) // 8
            else:       # no row wraps: the table of a step without tiling
                assert "wrap" not in lay and untiled
                assert host.numel() == 4 * Bc + lay["f32"][2] + lay["i32"][2]
            for q in plan.order:
                q.k += 1
            active = [q for q in active if q.k < q.steps]
    assert seen == {True, False}
