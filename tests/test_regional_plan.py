"""Regional prompts without a GPU: the oracle against the reference fixture, and the host table and its validation."""
import pytest
import torch

from helpers import load_golden, oracle_cfg, t


def _fixture():
    cfg, sd, g = load_golden("paella_tiny.npz")
    _, _, z = load_golden("regional_tiny.npz")
    base = [dict(byt5=t(g["byt5"][b:b + 1]), clip=t(g["clip"][b:b + 1]), clip_image=t(g["clip_image"][b:b + 1])) for b in range(2)]
    rp = [[{key: t(z[f"rp{b}{k}_{key}"]) for key in ("byt5", "clip", "clip_image") if f"rp{b}{k}_{key}" in z} for k in range(2)]
          for b in range(2)]
    return cfg, sd, g, z, base, rp


def test_oracle_matches_reference_fixture():
    from oracle import regional as orr
    cfg, sd, g, z, base, rp = _fixture()
    for n, x in ((8, t(g["x"])), (16, t(z["x16"]))):
        regs = [[t(z[f"reg{n}_{b}{k}"]) for k in range(2)] for b in range(2)]
        got = orr.paella_forward(sd, oracle_cfg(cfg), x, t(g["r"]), [[base[b]] + rp[b] for b in range(2)], orr.token_masks(regs, (n, n)))
        err = float((got - t(z[f"logits_{n}"])).abs().max())
        assert err < 1e-4, (n, err)
    # the masks matter: sample 0 without its regions is a different forward
    plain = orr.paella_forward(sd, oracle_cfg(cfg), t(g["x"]), t(g["r"]), [[base[b]] for b in range(2)],
                               torch.ones(2, 8, 8, dtype=torch.uint8))
    assert float((plain - t(z["logits_8"])).abs().max()) > 1e-2


def _inputs(L=3):
    return {"byt5": torch.randn(1, L, 8)}


def test_regional_table_layout():
    from paella_b200 import ops
    a = torch.zeros(4, 4, dtype=torch.bool)
    a[:, :2] = True
    b = torch.zeros(4, 4, dtype=torch.bool)
    b[1:3] = True
    p1, p2, p3 = _inputs(), _inputs(5), _inputs(2)
    masks, prompts = ops.regional_table([[(p1, a), (p2, b)], None, [(p3, torch.zeros(4, 4, dtype=torch.bool))]], 3, (4, 4))
    assert masks.dtype == torch.uint8 and masks.shape == (3, 4, 4)
    want0 = (a.to(torch.uint8) << 1) | (b.to(torch.uint8) << 2)
    want0[want0 == 0] = 1
    assert torch.equal(masks[0], want0)
    assert bool((masks[1] == 1).all()) and bool((masks[2] == 1).all())      # an empty region: every token in no region
    assert prompts[0] == [p1, p2] and prompts[1] == [] and prompts[2] == [p3]
    assert ops.regional_table(None, 2, (4, 4)) is None
    assert ops.regional_table([None, []], 2, (4, 4)) is None


@pytest.mark.parametrize("bad", [
    "x", [None], [[(None, None)]] * 2, [[(_inputs(),)], None],
    [[(_inputs(), torch.ones(4, 4, dtype=torch.bool))] * 8, None],
    [[(_inputs(), torch.ones(4, 5, dtype=torch.bool))], None],
    [[(_inputs(), torch.ones(4, 4))], None],
    [[({"byt5": torch.randn(2, 3, 8)}, torch.ones(4, 4, dtype=torch.bool))], None],
    [[({"byt5": torch.randn(1, 3, 8), "clip": torch.randn(2, 8)}, torch.ones(4, 4, dtype=torch.bool))], None],
    [[({"clip": torch.randn(1, 8)}, torch.ones(4, 4, dtype=torch.bool))], None],
    [(_inputs(), torch.ones(4, 4, dtype=torch.bool)), None],
], ids=["str", "short", "pair-of-none", "one-tuple", "eight-regions", "shape", "dtype", "batch-2-inputs", "batch-2-clip",
        "no-byt5", "unwrapped-pair"])
def test_regional_table_refuses(bad):
    from paella_b200 import ops
    with pytest.raises(ValueError):
        ops.regional_table(bad, 2, (4, 4))


def test_regions_with_attn_weights_refused():
    from paella_b200 import ops
    table = ops.regional_table([[(_inputs(), torch.ones(4, 4, dtype=torch.bool))], None], 2, (4, 4))
    ops.check_regions_unweighted(table, None)
    ops.check_regions_unweighted(table, [None, torch.ones(3)])
    with pytest.raises(ValueError):
        ops.check_regions_unweighted(table, [torch.ones(3), None])
    with pytest.raises(ValueError):
        ops.check_regions_unweighted(table, torch.ones(3))
