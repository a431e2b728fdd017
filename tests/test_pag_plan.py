"""Perturbed-attention guidance without a GPU: the fp64 oracle against the reference fixture, the argument validation and mask
table (ops.pag_table), the mix coefficients with and without CFG, the sampler's rows around sampling_conditional_steps, and the
ptxas reports of the new attention instances."""
import glob
import math
import os
import re

import numpy as np
import pytest
import torch

from helpers import load_golden, oracle_cfg, t

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY_CFG = dict(c_in=16, c_out=16, num_labels=64, c_r=64, patch_size=2, c_cond=32, c_hidden=[32, 64, 64], nhead=[-1, 4, 4],
                blocks=[1, 2, 1], level_config=["CT", "CTA", "CTA"], clip_embd=24, byt5_embd=40, clip_seq_len=4, kernel_size=3,
                dropout=0.1, self_attn=True)


# ------------------------------------------------------------------ oracle against the reference fixture
@pytest.fixture(scope="module")
def tiny():
    cfg, sd, g = load_golden("paella_tiny.npz")
    z = np.load(os.path.join(ROOT, "tests", "golden", "pag_tiny.npz"))
    return oracle_cfg(cfg), sd, g, {k: z[k] for k in z.files}


def _forward(tiny, x, blocks, weights=None, zero=False):
    from oracle import pag as op
    cfg, sd, g, _ = tiny
    byt5, clip, ci = t(g["byt5"]), t(g["clip"]), t(g["clip_image"])
    if zero:
        byt5, clip, ci = torch.zeros_like(byt5), torch.zeros_like(clip), torch.zeros_like(ci)
    return op.paella_forward_pag(sd, cfg, x, t(g["r"]), byt5, clip, ci, blocks=blocks, attn_weights=weights)


@pytest.mark.parametrize("case", ["deep", "all", "down", "attnw", "x16"])
def test_oracle_matches_the_reference_fixture(tiny, case):
    _, _, g, f = tiny
    n = int(f["n_blocks"])
    blocks = {"deep": list(f["deep"]), "all": list(range(n)), "down": [0], "attnw": list(range(n)), "x16": list(f["deep"])}[case]
    x = t(f["x16"]) if case == "x16" else t(g["x"])
    w = [t(f["attn_weights"])] * 2 if case == "attnw" else None
    got = _forward(tiny, x, [blocks, None], w)
    want = t(f[f"logits_{case}"])
    assert float((got - want).abs().max()) < 2e-4
    plain = t(f["logits_x16_plain"] if case == "x16" else f["logits_attnw_plain"] if case == "attnw" else f["logits_plain"])
    assert float((got[1] - plain[1]).abs().max()) < 2e-4           # sample 1 is not perturbed
    # the perturbation is visible in sample 0, except at the deepest level of an 8 x 8 grid: one position, whose diagonal is the map
    assert (float((want[0] - plain[0]).abs().max()) > 1e-3) == (case != "deep")


def test_oracle_mix_matches_the_fixture(tiny):
    from oracle import pag as op
    _, _, g, f = tiny
    lc = _forward(tiny, t(g["x"]), None)
    lp = _forward(tiny, t(g["x"]), [list(range(int(f["n_blocks"])))] * 2)
    lu = _forward(tiny, t(g["x"]), None, zero=True)
    s, c = float(f["scale"]), float(f["cfg"])
    # the fixture perturbs sample 0 only
    assert float((op.pag_mix(lc, lp, s, lu, c)[0] - t(f["mix_cfg"])[0]).abs().max()) < 2e-3
    assert float((op.pag_mix(lc, lp, s)[0] - t(f["mix_nocfg"])[0]).abs().max()) < 2e-3


def test_perturbed_core_without_conditioning_is_the_identity():
    from oracle import pag as op
    g = torch.Generator().manual_seed(0)
    q, k = torch.randn(1, 9, 16, generator=g), torch.randn(1, 9, 16, generator=g)
    v = torch.randn(1, 9, 16, generator=g)
    assert torch.allclose(op.perturbed_core(q, k, v, 2, 9), v, atol=1e-12)


# ------------------------------------------------------------------ ops.pag_table
def test_default_blocks_are_the_deepest_level():
    from paella_b200 import ops
    from paella_b200.lora import attn_blocks
    assert ops.pag_default_blocks(TINY_CFG) == [2, 3]
    from paella_b200.modules import Paella
    default = Paella(byt5_embd=2560)._cfg           # the default configuration: 44 AttnBlocks, 6 at the deepest level each way
    blocks = attn_blocks(default)
    deep = ops.pag_default_blocks(default)
    assert len(blocks) == 44 and deep == list(range(16, 28))
    assert all(blocks[i][0].startswith(("down_blocks.2.", "up_blocks.0.")) for i in deep)


def test_pag_table_layout():
    from paella_b200 import ops
    scales, masks = ops.pag_table([None, 2.0, (1.5, [0, 5]), 0.0, (0, [1])], 5, 6, [2, 3])
    assert scales == [0.0, 2.0, 1.5, 0.0, 0.0]
    assert masks.dtype == torch.int64 and masks.tolist() == [0, 0b1100, 0b100001, 0, 0]
    assert ops.pag_table([None, 0.0], 2, 6, [2]) is None and ops.pag_table(None, 2, 6, [2]) is None
    # bit 63 is a uint64 mask bit, stored in int64
    _, masks = ops.pag_table([(1.0, [63])], 1, 64, [0])
    assert masks.view(torch.int64).tolist() == [-(1 << 63)]
    scales, masks = ops.pag_table([[1, 2], None], 2, 6, forward=True)
    assert scales == [1.0, 0.0] and masks.tolist() == [0b110, 0]


@pytest.mark.parametrize("bad", [
    "x", [1.0], [1.0, 2.0, 3.0], [True, None], [float("nan"), None], [float("inf"), None], [(1.0, []), None], [(1.0, [1, 1]), None],
    [(1.0, [6]), None], [(1.0, [-1]), None], [(1.0, [True]), None], [(1.0, [1.5]), None], [(1.0, 3), None], [(1.0,), None],
    [(1.0, [1], 2), None], ["2.0", None],
])
def test_pag_table_rejects(bad):
    from paella_b200 import ops
    with pytest.raises(ValueError):
        ops.pag_table(bad, 2, 6, [2, 3])


def test_pag_table_rejects_regions_edits_sources_and_exact():
    from paella_b200 import ops
    regions = (None, [[], [("inputs", "region")]])
    assert ops.pag_table([1.0, None], 2, 6, [2], regions=regions) is not None
    with pytest.raises(ValueError, match="prompt_regions"):
        ops.pag_table([None, 1.0], 2, 6, [2], regions=regions)
    inj = ops.attention_source_table([None, (0, 2), None], 3, 4)
    assert ops.pag_table([None, None, 1.0], 3, 6, [2], inject=inj) is not None
    for b in (0, 1):
        entry = [None] * 3
        entry[b] = 1.0
        with pytest.raises(ValueError, match="edit or source"):
            ops.pag_table(entry, 3, 6, [2], inject=inj)
    with pytest.raises(ValueError, match="exact"):
        ops.pag_table([1.0], 1, 6, [2], exact=True)
    with pytest.raises(ValueError):
        ops.pag_table([1.0], 1, 65, [2])


# ------------------------------------------------------------------ mix coefficients
def test_coefficients_are_the_double_formula_rounded():
    from paella_b200 import ops
    for cfg, ws, s in [(8.0, [], 3.0), (4.5, [0.7, -0.3], 1.25), (1.0, [], 2.0), (3.3, [0.1], -0.6)]:
        want = [cfg + s, 1.0 - cfg * (1.0 + sum(ws))] + [cfg * w for w in ws] + [-s]
        assert ops.guidance_coefficients(cfg, ws, s) == [float(np.float32(v)) for v in want]
        assert math.isclose(sum(want), 1.0, abs_tol=1e-12)
    assert ops.guidance_coefficients(None, [], 2.5) == [3.5, -2.5]
    # without PAG the coefficients are those of the guidance-prompt mix
    assert ops.guidance_coefficients(8.0, [0.5]) == ops.guidance_coefficients(8.0, [0.5], 0.0)


def test_mix_table_rows_with_and_without_cfg():
    from paella_b200 import ops
    rows, coef = ops.guidance_mix_table([[0.5], [], []], [0, 1, 3], [4, 5, 7], [[8], [], []], [[2.0, 3.0, 4.0]] * 2,
                                        [0.0, 1.5, 2.0], [-1, 9, 10])
    assert rows.tolist() == [[0, 4, 8], [1, 5, 9], [3, 7, 10]]
    assert coef[1, 0].tolist() == ops.guidance_coefficients(2.0, [0.5])
    assert coef[0, 1].tolist() == ops.guidance_coefficients(3.0, [], 1.5)
    rows, coef = ops.guidance_mix_table([[], []], [0, 2], None, [[], []], [[None, None]], [1.0, 2.0], [3, 4])
    assert rows.tolist() == [[0, 3], [2, 4]]
    assert coef[0].tolist() == [[2.0, -1.0], [3.0, -2.0]]


# ------------------------------------------------------------------ ptxas: the new instances do not spill
def test_perturb_instances_do_not_spill():
    logs = [p for p in glob.glob(os.path.join(ROOT, "paella_b200", "csrc", "build", "attention*.ptxas.log"))]
    if not logs:
        pytest.skip("the library has not been built here")
    seen = 0
    for path in logs:
        fn = None
        for line in open(path):
            m = re.search(r"Compiling entry function '([^']+)'", line) or re.search(r"Function properties for (\S+)", line)
            if m:
                fn = m.group(1)
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m and fn and "perturb" in fn:
                seen += 1
                assert m.group(1) == "0" and m.group(2) == "0", (os.path.basename(path), fn, line.strip())
    assert seen >= 8 * 6, seen         # 8 flag combinations: the wgmma kernel and the mma.sync kernel at 5 head dims


# ------------------------------------------------------------------ SamplingEngine: admission and the step table
def _request(slot, steps, pag=None, terms=0, cfg=(8.0, 3.0), cond_steps=None, weighted=False):
    from paella_b200 import ops
    from paella_b200 import utils as U
    from paella_b200.engine import Request
    cond_steps = steps if cond_steps is None else cond_steps
    n_mix = min(steps, cond_steps)
    cfgs = U._cfg_schedule(cfg, 1, steps)
    params, r = U.sampling_schedule(1, steps, (1.0, 0.3), cfgs, 1.0, 0.0, always=True)
    tl = [({"byt5": torch.zeros(1, 2, 4)}, 0.25 * (j + 1)) for j in range(terms)] or None
    mix = None
    if cfgs is not None and (tl or pag):
        mix = torch.tensor([ops.guidance_coefficients(cfgs[i], [w for _, w in tl or []], pag[0] if pag else 0.0)
                            for i in range(n_mix)], dtype=torch.float32)
        params[:n_mix, 0, :2] = torch.tensor([1.0, 0.0])
    elif pag:
        mix = torch.tensor([ops.guidance_coefficients(None, [], pag[0])] * n_mix, dtype=torch.float32)
    q = Request(steps, steps - 1, cond_steps, cfgs is not None, params[:, 0], r[:, 0], terms=tl, mix_coef=mix, pag=pag,
                attn_weights=torch.ones(3) if weighted else None)
    q.slot, q.uncond_slot = slot, 100 + slot
    q.term_slot = [200 + 10 * slot + j for j in range(terms)]
    return q


def test_engine_step_table_with_pag_around_sampling_conditional_steps():
    from paella_b200.engine import build_step_plan, step_host_table
    qs = [_request(0, 4, pag=(2.0, 0b1100), terms=1), _request(1, 4), _request(2, 4, pag=(1.5, 0b11), cond_steps=2),
          _request(3, 4, pag=(3.0, 0b101), cfg=None, cond_steps=3), _request(4, 4, terms=2)]
    for step in range(4):
        for q in qs:
            q.k = step
        plan = build_step_plan(qs, 64)
        order, Bc, n_pairs = plan.order, len(plan.order), plan.n_pairs
        pert = [i for i, q in enumerate(order) if q.pag is not None and q.k < q.cond_steps]
        assert plan.perturbed == pert
        term_src = [i for i, q in enumerate(order[:n_pairs]) for _ in range(q.n_terms)]
        assert plan.tail.tolist() == list(range(n_pairs)) + term_src + pert
        assert plan.kv_slot.tolist() == [q.slot for q in order] + [q.uncond_slot for q in order[:n_pairs]] + \
            [s for q in order[:n_pairs] for s in q.term_slot] + [order[i].slot for i in pert]
        n_rows = Bc + plan.tail.numel()
        p0 = n_rows - len(pert)
        want_masks = [0] * p0 + [order[i].pag[1] for i in pert]
        assert plan.pag_rows.tolist() == want_masks
        assert plan.pag_w_row.tolist() == [q.slot for q in order] + [64] * (p0 - Bc) + [order[i].slot for i in pert]
        t = Bc + n_pairs
        for y, i in enumerate(plan.composed):
            q = order[i]
            if i < n_pairs:
                want = [i, Bc + i] + list(range(t, t + q.n_terms)) + ([p0 + pert.index(i)] if i in pert else [])
                t += q.n_terms
                assert plan.params[i, 0] == 1.0 and plan.params[i, 1] == 0.0
            else:
                want = [i, p0 + pert.index(i)]
                assert q.guided is False
            assert plan.mix_rows[y, :len(want)].tolist() == want and bool((plan.mix_rows[y, len(want):] == -1).all())
            assert torch.equal(plan.mix_coef[y, :len(want)], q.mix_coef[q.k])
            assert abs(float(q.mix_coef[q.k].double().sum()) - 1.0) < 1e-5
        host, lay = step_host_table(plan, [0, 0] * Bc, [0, 0] * Bc)
        assert ("pag" in lay) == bool(pert) and ("w_row" in lay) == bool(pert)
        if pert:
            _, o, n = lay["pag"]
            assert host[o:o + n].tolist() == want_masks
            i32 = host[lay["i32"][1]:lay["i32"][1] + lay["i32"][2]].view(torch.int32)
            _, o, n = lay["w_row"]
            assert torch.equal(i32[o:o + n], plan.pag_w_row)
    # step 3: request 2 (cond_steps 2) and request 3 (cond_steps 3) are no longer perturbed; request 0 is
    assert [plan.order[i].slot for i in plan.perturbed] == [0]


def test_engine_step_table_without_pag_is_unchanged():
    from paella_b200.engine import build_step_plan, step_host_table
    qs = [_request(0, 3, terms=2), _request(1, 3), _request(2, 3, cfg=None)]
    plan = build_step_plan(qs, 64)
    assert plan.perturbed == [] and plan.composed == [0] and plan.mix_rows.shape == (1, 4)
    _, lay = step_host_table(plan, [0, 0] * 3, [0, 0] * 3)
    assert "pag" not in lay and "w_row" not in lay


# ------------------------------------------------------------------ every kernel that existed before PAG keeps its SASS
def test_existing_kernels_keep_their_sass():
    """tests/golden/sass_before_pag.json holds the SHA-1 of every kernel's SASS (cuobjdump -sass, per function) in the library
    built without perturbed-attention guidance, with the nvcc release that built it.  Adding the _perturb instances and the
    PERTURB template parameter must leave every one of them identical: the plain paths run the same code."""
    import hashlib
    import json
    import shutil
    import subprocess
    so = os.path.join(ROOT, "paella_b200", "libpaella_b200.so")
    if shutil.which("cuobjdump") is None or shutil.which("nvcc") is None or not os.path.exists(so):
        pytest.skip("cuobjdump, nvcc or the built library is not available")
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_before_pag.json")))
    ver = subprocess.run(["nvcc", "--version"], capture_output=True, text=True, check=True).stdout
    if want["nvcc"] not in ver:
        pytest.skip(f"the reference hashes come from nvcc {want['nvcc']}")
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    got, fn, buf = {}, None, []
    for line in out.splitlines() + ["Function : <end>"]:
        m = re.search(r"Function : (\S+)", line)
        if m:
            if fn:
                got[fn] = hashlib.sha1("\n".join(buf).encode()).hexdigest()
            fn, buf = m.group(1), []
        elif fn:
            buf.append(line)
    changed = [k for k, h in want["functions"].items() if got.get(k) != h]
    assert not changed, changed[:5]
    assert all("perturb" in k for k in got if k not in want["functions"])
