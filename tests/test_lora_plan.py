"""LoRA adapters on the CPU: the oracle against the reference fixture, merge_lora against the oracle, the adapter format's
validation, the alpha / r scaling, the packed blob layout, and the per-sample table (no GPU needed)."""
import math
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN, load_golden, oracle_cfg, t
from oracle import lora as ol
from oracle import paella_oracle as po
from paella_b200 import ops
from paella_b200.lora import attn_blocks, load_lora, merge_lora, pack_lora, parse_lora, served_targets, unpack_lora

TOL = dict(rtol=2e-4, atol=2e-5)


def _fixture():
    cfg, sd, _ = load_golden("paella_tiny.npz")
    z = np.load(os.path.join(GOLDEN, "lora_tiny.npz"))
    la = {k[2:]: torch.from_numpy(z[k].copy()) for k in z.files if k.startswith("a:")}
    lb = {k[2:]: torch.from_numpy(z[k].copy()) for k in z.files if k.startswith("b:")}
    return cfg, sd, z, la, lb


@pytest.fixture(scope="module")
def tiny_cpu():
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).eval()
    m.load_state_dict(sd)
    return m, cfg, sd


def test_fixture_adapters_are_not_vacuous():
    _, _, z, la, lb = _fixture()
    assert all(float(v.abs().max()) > 0 for k, v in list(la.items()) + list(lb.items()) if k.endswith("lora_B.weight"))
    d = np.abs(z["logits"] - z["logits_base"]).reshape(4, -1).max(1)
    assert d[0] > 0.14 and d[2] > 0.14 and d[3] > 0.14 and d[1] < 1e-4


def test_oracle_on_merged_weights_reproduces_reference_fixture():
    cfg, sd, z, la, lb = _fixture()
    oc = oracle_cfg(cfg)
    adapters = {0: la, 1: lb}
    for i in range(4):
        w = int(z["which"][i])
        msd = sd if w < 0 else ol.merge(sd, adapters[w], float(z["scales"][i]))
        got = po.paella_forward(msd, oc, t(z["x"][i:i + 1]), t(z["r"][i:i + 1]), t(z["byt5"][i:i + 1]), t(z["clip"][i:i + 1]))
        torch.testing.assert_close(got, t(z["logits"][i:i + 1]), **TOL)


def test_merge_lora_matches_oracle_and_alpha_over_r():
    cfg, sd, _, la, lb = _fixture()
    for lsd, s in ((la, 1.0), (lb, 0.5), (lb, -1.25)):
        got, want = merge_lora(sd, lsd, scale=s), ol.merge(sd, lsd, s)
        assert got.keys() == want.keys()
        for k in got:
            torch.testing.assert_close(got[k], want[k], rtol=0, atol=0)
    # alpha / r: b has alpha 8 at rank 16 -> half the delta of the same adapter without alpha
    m = "down_blocks.1.3.kv_mapper.1"
    no_alpha = {k: v for k, v in lb.items() if not k.endswith(".alpha")}
    d8 = merge_lora(sd, lb)[m + ".weight"].double() - sd[m + ".weight"].double()
    d16 = merge_lora(sd, no_alpha)[m + ".weight"].double() - sd[m + ".weight"].double()
    torch.testing.assert_close(d8, 0.5 * d16, rtol=1e-5, atol=1e-7)
    exp = 0.5 * lb[m + ".lora_B.weight"].double() @ lb[m + ".lora_A.weight"].double()
    torch.testing.assert_close(d8, exp, rtol=1e-5, atol=1e-7)


def test_merge_lora_other_targets_and_in_proj():
    cfg, sd, _, _, _ = _fixture()
    g = torch.Generator().manual_seed(3)
    lsd = {"down_blocks.1.1.channelwise.0.lora_A.weight": torch.randn(2, 64, generator=g),      # ResBlock MLP (Linear)
           "down_blocks.1.1.channelwise.0.lora_B.weight": torch.randn(256, 2, generator=g),
           "clf.1.lora_A.weight": torch.randn(2, 32, generator=g), "clf.1.lora_B.weight": torch.randn(64, 2, generator=g),  # 1x1 conv
           "up_blocks.1.2.attention.attn.in_proj.lora_A.weight": torch.randn(2, 64, generator=g),
           "up_blocks.1.2.attention.attn.in_proj.lora_B.weight": torch.randn(192, 2, generator=g)}
    got = merge_lora(sd, lsd, 0.3)
    assert got["clf.1.weight"].shape == sd["clf.1.weight"].shape
    d = got["up_blocks.1.2.attention.attn.in_proj_weight"].double() - sd["up_blocks.1.2.attention.attn.in_proj_weight"].double()
    want = 0.3 * lsd["up_blocks.1.2.attention.attn.in_proj.lora_B.weight"].double() @ lsd["up_blocks.1.2.attention.attn.in_proj.lora_A.weight"].double()
    torch.testing.assert_close(d, want, rtol=1e-5, atol=1e-6)
    bad = {"down_blocks.1.0.1.lora_A.weight": torch.randn(2, 128), "down_blocks.1.0.1.lora_B.weight": torch.randn(64, 2)}
    with pytest.raises(ValueError, match="not a Linear or 1x1-conv"):
        merge_lora(sd, bad)
    with pytest.raises(ValueError, match="finite"):
        merge_lora(sd, lsd, float("nan"))


def _one(mod="down_blocks.1.3.attention.attn.out_proj", r=4, fin=64, fout=64):
    return {f"{mod}.lora_A.weight": torch.randn(r, fin), f"{mod}.lora_B.weight": torch.randn(fout, r)}


@pytest.mark.parametrize("case, match", [
    ("mlp", "merge_lora"),
    ("timestep", "merge_lora"),
    ("embedding", "merge_lora"),
    ("out_mapper", "merge_lora"),
    ("unknown_module", "unknown key"),
    ("unknown_suffix", "unknown key"),
    ("shape", "expected"),
    ("a_without_b", "lora_B.weight' is missing"),
    ("rank_0", "rank 0"),
    ("rank_65", "rank 65"),
    ("mixed_rank", "one rank per adapter"),
    ("nan", "non-finite"),
])
def test_load_lora_rejects(tiny_cpu, case, match):
    m, _, _ = tiny_cpu
    sd = {
        "mlp": lambda: _one("down_blocks.1.1.channelwise.0", 4, 64, 256),
        "timestep": lambda: _one("down_blocks.1.2.mapper", 4, 64, 128),
        "embedding": lambda: _one("embedding.1", 4, 64, 32),
        "out_mapper": lambda: _one("out_mapper.1", 4, 16, 64),
        "unknown_module": lambda: _one("down_blocks.1.9.attention.attn.out_proj"),
        "unknown_suffix": lambda: {**_one(), "down_blocks.1.3.attention.attn.out_proj.lora_C.weight": torch.zeros(1)},
        "shape": lambda: _one(fin=32),
        "a_without_b": lambda: {"down_blocks.1.3.kv_mapper.1.lora_A.weight": torch.randn(4, 32)},
        "rank_0": lambda: _one(r=0),
        "rank_65": lambda: _one(r=65),
        "mixed_rank": lambda: {**_one(), **_one("down_blocks.1.6.attention.attn.out_proj", r=8)},
        "nan": lambda: {**_one(), "down_blocks.1.3.attention.attn.out_proj.lora_B.weight": torch.full((64, 4), math.nan)},
    }[case]()
    with pytest.raises(ValueError, match=match):
        load_lora(m, sd)


def test_pack_unpack_round_trip_with_row_sums():
    cfg, _, _, la, lb = _fixture()
    for lsd, rank, alpha in ((la, 4, 4.0), (lb, 16, 8.0)):
        mods, r = parse_lora(lsd)
        assert r == rank
        blob, targets = pack_lora(cfg, mods, r)
        assert blob.dtype == torch.uint8 and blob.numel() % 256 == 0
        served = served_targets(cfg)
        assert len(targets) == len(attn_blocks(cfg)) == 6
        assert sum(bin(b).count("1") for b in targets) == len(mods)
        got = unpack_lora(cfg, blob, r, targets)
        assert sorted(got) == sorted(mods)
        rp = (r + 7) // 8 * 8
        for mod, (a16, b16, aux) in got.items():
            a, b, al = mods[mod]
            _, _, fin, fout = served[mod]
            assert a16.shape == (rp, fin) and b16.shape == (fout, rp) and aux.shape == (rp + 1,)
            assert torch.equal(a16[:r], a.half()) and not a16[r:].any()
            assert torch.equal(b16[:, :r], b.half()) and not b16[:, r:].any()
            assert torch.equal(aux[:rp], a16.double().sum(1).float())
            assert float(aux[rp]) == pytest.approx(alpha / r) and al == alpha


def test_blob_size_per_rank_on_default_model():
    """About 0.88 MB per rank on the default model: 44 AttnBlocks x r x 9,984 fp16 values (in_proj 4c, out_proj 2c, kv_mapper
    c_cond + c), plus the row sums and padding."""
    from paella_b200.modules import Paella
    with torch.device("meta"):
        cfg = Paella()._cfg
    blocks = attn_blocks(cfg)
    assert len(blocks) == 44 and all(c == 1280 for _, c in blocks)
    g = torch.Generator().manual_seed(0)
    mods = {}
    for pre, c in blocks:
        for name, (k, bit, fin, fout) in served_targets(cfg).items():
            if name.startswith(pre + "."):
                mods[name] = (torch.randn(16, fin, generator=g), torch.randn(fout, 16, generator=g), 16.0)
    blob, _ = pack_lora(cfg, mods, 16)
    assert abs(blob.numel() - 44 * 16 * 9984 * 2) / (44 * 16 * 9984 * 2) < 0.01


def test_lora_table(tiny_cpu):
    m, cfg, _ = tiny_cpu
    _, _, _, la, lb = _fixture()
    a, b = load_lora(m, la), load_lora(m, lb)
    assert a.rank == 4 and b.rank == 16 and a.targets == [7] * 6
    assert ops.lora_table(None, 3, m) is None
    assert ops.lora_table([None, (a, 0.0), None], 3, m) is None          # scale 0 is no adapter
    ads, ids, sc = ops.lora_table([a, None, (b, 0.5), (a, 2)], 4, m)
    assert ads[0] is a and ads[1] is b and len(ads) == 2
    assert ids.tolist() == [0, -1, 1, 0] and sc.tolist() == [1.0, 0.0, 0.5, 2.0]
    ads, ids, sc = ops.lora_table((b, 0.25), 3, m)
    assert ads == [b] and ids.tolist() == [0, 0, 0] and sc.tolist() == [0.25] * 3
    assert ops.lora_entries(ops.lora_table([a, None], 2, m), 2) == [(a, 1.0), None]
    for bad, match in (([a], "1 entries"), ([a, "x"], "expected None"), ([(a, math.inf), None], "finite"),
                       ([(a, True), None], "real number"), ("a", "expected None")):
        with pytest.raises(ValueError, match=match):
            ops.lora_table(bad, 2, m)
    from paella_b200.modules import Paella
    other = Paella(**{**cfg, "c_cond": 40})
    with pytest.raises(ValueError, match="another model configuration"):
        ops.lora_table(a, 2, other)
    many = [load_lora(m, la) for _ in range(33)]
    with pytest.raises(ValueError, match="33 distinct"):
        ops.lora_table(many, 33, m)


def test_engine_step_host_table_with_adapters(tiny_cpu):
    """The step table carries each row's adapter index into the step's distinct adapters and its scale, in the step's row order
    (guided first), only when some row has an adapter; a step without one is laid out exactly as before."""
    from paella_b200 import utils as U
    from paella_b200.engine import Request, build_step_plan, step_host_table
    m, _, _ = tiny_cpu
    _, _, _, la, lb = _fixture()
    a, b = load_lora(m, la), load_lora(m, lb)

    def req(slot, guided, lora):
        cfgs = U._cfg_schedule((8.0, 8.0) if guided else None, 1, 4)
        params, r = U.sampling_schedule(1, 4, (1.0, 0.5), cfgs, 1.0, 0.0, always=True)
        q = Request(4, 3, 4, guided, params[:, 0], r[:, 0], lora=lora)
        q.slot, q.uncond_slot = slot, 10 + slot
        return q
    plain = [req(0, True, None), req(1, False, None), req(2, True, None)]
    host0, lay0 = step_host_table(build_step_plan(plain), [0, 0] * 3, [0, 0] * 3)
    assert "lora_id" not in lay0 and "lora_scale" not in lay0
    active = [req(0, False, (b, 0.5)), req(1, True, None), req(2, True, (a, 2.0)), req(3, False, (a, 1.0)), req(4, True, (b, -1.0))]
    plan = build_step_plan(active)
    assert [q.slot for q in plan.order] == [1, 2, 4, 0, 3]
    assert plan.loras and plan.adapters[0] is a and plan.adapters[1] is b
    assert plan.lora_id.tolist() == [-1, 0, 1, 1, 0] and plan.lora_scale.tolist() == [0.0, 2.0, -1.0, 0.5, 1.0]
    host, lay = step_host_table(plan, [0, 0] * 5, [0, 0] * 5)
    f32 = host[lay["f32"][1]:lay["f32"][1] + lay["f32"][2]].view(torch.float32)
    i32 = host[lay["i32"][1]:lay["i32"][1] + lay["i32"][2]].view(torch.int32)
    _, o, n = lay["lora_id"]
    assert i32[o:o + n].tolist() == plan.lora_id.tolist()
    _, o, n = lay["lora_scale"]
    assert f32[o:o + n].tolist() == plan.lora_scale.tolist()
    # the rest of the table is where it was
    base = build_step_plan([req(q.slot, q.guided, None) for q in active])
    _, lay_b = step_host_table(base, [0, 0] * 5, [0, 0] * 5)
    for k in ("r", "params", "t_next", "row_slot", "kv_slot"):
        assert lay[k] == lay_b[k]


def test_engine_admission_keeps_adapters_in_flight_within_the_launch_limit(tiny_cpu):
    """With max_batch above 32 and more distinct adapters queued than one step's launches take, admission holds the request whose
    adapter would be the 33rd in flight (and everything behind it, FIFO) until a request retires; every request is admitted in the
    end, and no step plan holds more than 32 distinct adapters."""
    import collections
    import random

    from paella_b200 import utils as U
    from paella_b200.engine import Request, admit_from_queue, build_step_plan
    m, _, _ = tiny_cpu
    _, _, _, la, _ = _fixture()
    adapters = [load_lora(m, la) for _ in range(40)]
    rng = random.Random(0)

    def req(i):
        steps = rng.choice([1, 2, 3])
        params, r = U.sampling_schedule(1, steps, (1.0, 0.5), U._cfg_schedule((8.0, 8.0), 1, steps), 1.0, 0.0, always=True)
        lora = None if i % 10 == 9 else (adapters[i % 40], 1.0)
        q = Request(steps, steps - 1, steps, True, params[:, 0], r[:, 0], lora=lora)
        q.name = i
        return q
    queue = collections.deque(req(i) for i in range(60))
    free, active, admitted, held = list(range(48)), [], [], 0
    for _ in range(200):
        new = admit_from_queue(queue, len(free), active)
        for q in new:
            q.slot = free.pop(0)
            q.uncond_slot = 100 + q.slot
        active += new
        admitted += [q.name for q in new]
        if not active and not queue:
            break
        plan = build_step_plan(active)
        assert len(plan.adapters) <= ops.MAX_LORA_ADAPTERS
        if queue and len(free) > 0:      # a free slot and a request left behind: held for its adapter
            assert len(ops.distinct_adapters([q.lora for q in active] + [queue[0].lora])) > ops.MAX_LORA_ADAPTERS
            held += 1
        for q in active:
            q.k += 1
        free += [q.slot for q in active if q.k == q.steps]
        active = [q for q in active if q.k < q.steps]
    assert admitted == list(range(60)) and held > 0
    assert len(ops.distinct_adapters([(a, 1.0) for a in adapters])) == 40
