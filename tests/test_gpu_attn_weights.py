"""Per-sample attn_weights: one post-softmax weight vector per sample (Paella.features / forward, sample_notebook,
SamplingEngine), so notebook-style requests whose prompts, and so whose vectors, differ share one batch.

  * an all-equal table gives the single-vector call's features, logits and tokens, bit for bit (tiny and default model)
  * in a heterogeneous batch, row i equals row i of the single-vector call with vector i, bit for bit: varlen conditioning
    with and without clip / clip_image, a shared unconditional slot, a None row, a vector of length 1, one that crosses a
    64-key chunk boundary and one longer than the conditioning that reaches into the self keys.  Tiny model (mma.sync
    kernel) in process; the default model (head_dim 80: the wgmma kernel) in a child process, and again in a child
    process with PB200_ATTN_MMA_SYNC=1
  * tiny model: rows equal batch-1 sample_notebook calls with per-sample generators; each sample matches the CPU oracle
  * the unconditional tail of a guided step is never weighted
  * SamplingEngine with per-request weights and intermediates equals batch-1 sample_notebook runs (tiny model, and the
    default model with one forced GEMM tile width in a child process); no host synchronisation in submit or step
  * every ValueError is raised before any generator moves
"""
import os
import subprocess
import sys

import pytest
import torch

from helpers import load_golden, log_jsonl, oracle_cfg

pytestmark = pytest.mark.gpu
DEV = "cuda"
MAX_ABS, RMS = 7e-3, 1.2e-3             # the tiny golden model's bounds of tests/test_gpu_model.py


def _log(payload):
    log_jsonl("attn_weights.jsonl", payload)


def _gens(seeds):
    return [torch.Generator(device=DEV).manual_seed(s) for s in seeds]


def _vec(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, generator=g) * 1.6 + 0.2


def _notebook_vec(n):
    """paella_inference.ipynb cell 7: 1.2 everywhere, 0.4 on the last 4 entries."""
    v = torch.full((n,), 1.2)
    v[-4:] = 0.4
    return v


def _inputs(m, B, L, clip=True, clip_image=False, seed=0, zeros=False):
    g = torch.Generator().manual_seed(seed)
    E, C = m.byt5_mapper.in_features, m.clip_mapper.in_features
    d = {"byt5": torch.randn(B, L, E, generator=g)}
    if clip:
        d["clip"] = torch.randn(B, C, generator=g)
    if clip_image:
        d["clip_image"] = torch.randn(B, C, generator=g)
    if zeros:
        d = {k: torch.zeros_like(v) for k, v in d.items()}
    return {k: v.to(DEV) for k, v in d.items()}


def _row(d, i):
    return {k: v[i:i + 1] for k, v in d.items()}


@pytest.fixture(scope="module")
def tiny():
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    return m, cfg, sd


def _default_model():
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    return m.to(DEV)


# ------------------------------------------------------------------ weighted rows
def _heterogeneous_case(m, H):
    """Varlen conditioning groups of one sample each plus a shared all-zero unconditional group, and one vector per sample:
    a long one crossing a 64-key chunk boundary, None, length 1, and one longer than the conditioning (into the self keys)."""
    specs = [(72, True, True), (9, True, False), (5, False, False), (13, False, True)]
    groups = [_inputs(m, 1, L, c, ci, seed=10 + i) for i, (L, c, ci) in enumerate(specs)]
    B = len(groups)
    lens = [m.conditioning_seq_len(g) for g in groups]
    # 40 keys end 80 conditioning rows: they cross key 64 of the mma.sync kernel's walk over [self ; cond] at every level,
    # and the wgmma kernel's conditioning chunk boundary (self keys + 64) at the 16-position level
    vecs = [_vec(40, 1), None, _vec(1, 2), _vec(lens[3] + 3, 3)]
    for i, v in enumerate(vecs):
        assert v is None or v.numel() <= m.max_attn_weights((H, H), lens[i])
    uncond = _inputs(m, B, 6, True, False, zeros=True)
    return groups, uncond, vecs


def _check_heterogeneous_rows(m, H, tag):
    from paella_b200 import ops
    groups, uncond, vecs = _heterogeneous_case(m, H)
    B = len(groups)
    with torch.inference_mode():
        cond = m.prepare_conditioning(groups + [uncond], (H, H))
        assert cond.slots == B + 1                      # the unconditional rows share one slot
        x = torch.randint(0, m.num_labels, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
        r = torch.rand(B, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
        table, lens = ops.attn_weights_table(vecs, B, [10 ** 6] * B)
        w_d, len_d = ops.attn_weights_to_device(table, lens, DEV)
        got = m.features(x, r, cond, w_d, B, cfg_pairs=True, w_len=len_d)
        n = H * H
        for i, v in enumerate(vecs):
            want = m.features(x, r, cond, v.to(DEV) if v is not None else None, B if v is not None else 0, cfg_pairs=True)
            assert torch.equal(got[i * n:(i + 1) * n], want[i * n:(i + 1) * n]), f"{tag}: conditional row {i}"
            assert torch.equal(got[(B + i) * n:(B + i + 1) * n], want[(B + i) * n:(B + i + 1) * n]), f"{tag}: unconditional row {i}"
        # a None row is the unweighted call's row
        plain = m.features(x, r, cond, cfg_pairs=True)
        assert torch.equal(got[n:2 * n], plain[n:2 * n])
        assert not torch.equal(got[:n], plain[:n]), "the weighted row must differ from the unweighted one"
    _log({"test": "heterogeneous_rows", "model": tag})


def _check_all_equal(m, H, tag, steps=3):
    """An all-equal table gives the single-vector call, bit for bit: logits of forward and sample_notebook tokens."""
    from paella_b200 import utils as U
    B, L = 3, 20
    cond = _inputs(m, B, L, True, True, seed=1)
    uncond = _inputs(m, B, L, True, True, zeros=True)
    v = _notebook_vec(L)
    x = torch.randint(0, m.num_labels, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    r = torch.full((B,), 0.6, device=DEV)
    with torch.inference_mode():
        one = m(x, r, **cond, attn_weights=v.to(DEV))
        per = m(x, r, **cond, attn_weights=[v] * B)
    assert torch.equal(one, per), f"{tag}: forward logits"
    for gen in (None, "list"):
        outs = []
        for aw in (v.to(DEV), [v] * B):
            torch.manual_seed(7)
            g = _gens([1, 2, 3]) if gen else None
            outs.append(U.sample_notebook(m, cond, (B, H, H), uncond, steps=steps, attn_weights=aw, generator=g))
        (ta, ia), (tb, ib) = outs
        assert torch.equal(ta, tb) and len(ia) == len(ib) and all(torch.equal(a, b) for a, b in zip(ia, ib)), f"{tag}: tokens"
    _log({"test": "all_equal", "model": tag})


def test_tiny_all_equal_table_equals_single_vector(tiny):
    _check_all_equal(tiny[0], 8, "tiny")


def test_tiny_heterogeneous_rows_equal_single_vector_calls(tiny):
    _check_heterogeneous_rows(tiny[0], 16, "tiny")


def test_tiny_rows_equal_batch1_notebook_calls(tiny):
    """Per-sample generators: row i equals the batch-1 sample_notebook call with vector i, tokens, intermediates and offsets."""
    from paella_b200 import utils as U
    m, H, B, L = tiny[0], 8, 4, 11
    cond = _inputs(m, B, L, True, False, seed=3)
    uncond = _inputs(m, B, L, True, False, zeros=True)
    S = m.conditioning_seq_len(cond)
    vecs = [_notebook_vec(L), None, _vec(1, 4), _vec(S + 1, 5)]       # S + 1: every key of the deepest AttnBlock
    kw = dict(steps=4, renoise_steps=2, cfg=(7.0, 3.0), sampling_conditional_steps=3, temperature=(0.9, 0.4))
    gens = _gens([11, 12, 13, 14])
    toks, inter = U.sample_notebook(m, cond, (B, H, H), uncond, attn_weights=vecs, generator=gens, **kw)
    for i, v in enumerate(vecs):
        g = _gens([11 + i])
        t1, i1 = U.sample_notebook(m, _row(cond, i), (1, H, H), _row(uncond, i), attn_weights=v, generator=g, **kw)
        assert torch.equal(toks[i:i + 1], t1), f"row {i}"
        assert all(torch.equal(a[i:i + 1], b) for a, b in zip(inter, i1)) and len(inter) == len(i1)
        assert g[0].get_offset() == gens[i].get_offset()


def test_tiny_each_sample_matches_the_oracle(tiny):
    from oracle.paella_oracle import paella_forward
    m, cfg, sd = tiny
    H, B, L = 8, 3, 7
    cond = _inputs(m, B, L, True, True, seed=6)
    S = m.conditioning_seq_len(cond)
    vecs = [_notebook_vec(L), _vec(S + 1, 7), None]
    x = torch.randint(0, m.num_labels, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(8))
    r = torch.tensor([0.9, 0.5, 0.2], device=DEV)
    with torch.inference_mode():
        got = m(x, r, **cond, attn_weights=vecs).cpu()
    sd = {k: v.float().cpu() for k, v in sd.items()}
    for i, v in enumerate(vecs):
        want = paella_forward(sd, oracle_cfg(cfg), x[i:i + 1].cpu(), r[i:i + 1].cpu(), cond["byt5"][i:i + 1].cpu(),
                              cond["clip"][i:i + 1].cpu(), cond["clip_image"][i:i + 1].cpu(), attn_weights=v)
        d = got[i:i + 1] - want
        mx, rms = float(d.abs().max()), float(d.pow(2).mean().sqrt())
        _log({"test": "oracle", "row": i, "max_abs": mx, "rms": rms})
        assert mx < MAX_ABS and rms < RMS, (i, mx, rms)


def test_tiny_unconditional_tail_is_unweighted(tiny):
    """A guided step's rows: the cfg mix of the weighted conditional forward and the unweighted unconditional forward."""
    from paella_b200 import ops
    from paella_b200 import utils as U
    m, H, B, L = tiny[0], 8, 3, 9
    cond = _inputs(m, B, L, True, False, seed=9)
    uncond = _inputs(m, B, L, True, False, zeros=True)
    vecs = [_notebook_vec(L), _vec(3, 10), None]
    cfg, T = 6.0, 0.8
    init = ops.randint(m.num_labels, (B, H, H), DEV, torch.Generator(device=DEV).manual_seed(3))
    with torch.inference_mode():
        r = torch.ones(B, device=DEV)
        lc = m(init, r, **cond, attn_weights=vecs)
        lu = m(init, r, **uncond)
        want = ops.resample_logits(lc, lu, cfg, float(torch.linspace(T, T, 1)[0]), "argmax")
    g = torch.Generator(device=DEV).manual_seed(3)
    toks, _ = U.sample_notebook(m, cond, (B, H, H), uncond, steps=1, temperature=(T, T), cfg=(cfg, cfg), mode="argmax",
                                attn_weights=vecs, generator=g)
    assert torch.equal(toks, want)


# ------------------------------------------------------------------ default model (head_dim 80), child processes
@pytest.mark.skipif(not os.environ.get("PB200_ATTN_W_CHILD"), reason="run in a child process")
def test_default_weighted_rows_child():
    m = _default_model()
    _check_all_equal(m, 16, "default", steps=2)
    _check_heterogeneous_rows(m, 16, "default")


def _child(test, env):
    here = os.path.dirname(os.path.abspath(__file__))
    p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.join(here, os.path.basename(__file__)),
                        "-k", test], env=dict(os.environ, **env), capture_output=True, text=True, timeout=1200,
                       cwd=os.path.dirname(here))
    assert p.returncode == 0 and "1 passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


@pytest.mark.parametrize("kernel", ["wgmma", "mma_sync"])
def test_default_weighted_rows(kernel):
    env = {"PB200_ATTN_W_CHILD": "1"}
    if kernel == "mma_sync":
        env["PB200_ATTN_MMA_SYNC"] = "1"
    _child("test_default_weighted_rows_child", env)


# ------------------------------------------------------------------ SamplingEngine
def _reference(m, spec, H):
    from paella_b200 import utils as U
    g = torch.Generator(device=DEV).manual_seed(spec["seed"])
    kw = {k: spec[k] for k in ("steps", "renoise_steps", "temperature", "cfg", "t_start", "t_end", "sampling_conditional_steps")
          if k in spec}
    toks, inter = U.sample_notebook(m, spec["inputs"], (1, H, H), spec.get("uncond_ref"), init_x=spec.get("init_x"),
                                    attn_weights=spec.get("w"), generator=[g], **kw)
    return toks, inter, g.get_offset()


def _engine_schedule(m, H, L0=9):
    shared = _inputs(m, 1, 6, clip=True, zeros=True)
    inp = lambda L, c, ci, s: _inputs(m, 1, L, c, ci, seed=s)       # noqa: E731
    S = {}
    a_in, c_in = inp(L0, True, True, 20), inp(12, True, False, 22)
    S[0] = [dict(name="a", seed=1, steps=3, cfg=(8.0, 8.0), inputs=a_in, uncond_ref=shared, w=_notebook_vec(L0)),
            dict(name="b", seed=2, steps=5, cfg=None, inputs=inp(4, False, True, 21)),
            dict(name="c", seed=3, steps=2, cfg=(9.0, 2.0), sampling_conditional_steps=1, inputs=c_in, uncond_ref=shared,
                 w=_vec(m.max_attn_weights((H, H), m.conditioning_seq_len(c_in)), 4))]
    # queued behind the full engine: d takes c's slot with a shorter vector, e takes a's slot with none
    S[1] = [dict(name="d", seed=4, steps=4, cfg=(5.0, 5.0), renoise_steps=1, inputs=inp(3, True, False, 23),
                 uncond=inp(3, True, False, 24), uncond_ref=inp(3, True, False, 24), w=_vec(2, 5)),
            dict(name="e", seed=5, steps=3, cfg=(7.0, 3.0), sampling_conditional_steps=2, inputs=inp(7, False, False, 25),
                 uncond_ref=shared)]
    S[4] = [dict(name="f", seed=6, steps=2, cfg=None, temperature=(0.5, 0.5), inputs=inp(2, True, False, 26), w=_vec(1, 6))]
    return S, shared


def _run_engine(eng, S, sync_check=False):
    subs, step = [], 0
    while step <= max(S) or eng.busy:
        for spec in S.get(step, []):
            kw = {k: spec[k] for k in ("steps", "renoise_steps", "temperature", "cfg", "t_start", "t_end",
                                       "sampling_conditional_steps", "init_x") if k in spec}
            g = torch.Generator(device=DEV).manual_seed(spec["seed"])
            subs.append((spec, eng.submit(spec["inputs"], spec.get("uncond"), generator=g, attn_weights=spec.get("w"),
                                          keep_intermediates=True, **kw), g))
        eng.step()
        step += 1
    return subs


def _check_engine(m, subs, H):
    for spec, req, g in subs:
        assert req.done
        toks, inter, off = _reference(m, spec, H)
        assert torch.equal(req.result, toks), f"request {spec['name']}: tokens"
        assert len(req.intermediates) == len(inter) and all(torch.equal(a, b) for a, b in zip(req.intermediates, inter)), \
            f"request {spec['name']}: intermediates"
        assert g.get_offset() == off, f"request {spec['name']}: generator offset"


def test_tiny_engine_weighted_requests_equal_batch1_notebook_runs(tiny):
    from paella_b200.engine import SamplingEngine
    m, H = tiny[0], 8
    S, shared = _engine_schedule(m, H)
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=3, max_cond_len=20, unconditional_inputs=shared)
    subs = _run_engine(eng, S)
    slots = {spec["name"]: req.slot for spec, req, _ in subs}
    assert slots["d"] == slots["c"] and slots["e"] == slots["a"], slots       # the reused slots of the scenario
    _check_engine(m, subs, H)
    _log({"test": "tiny_engine", "requests": len(subs)})


def test_engine_with_weights_does_not_synchronise(tiny):
    from paella_b200.engine import SamplingEngine
    m, H = tiny[0], 8
    S, shared = _engine_schedule(m, H)
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=3, max_cond_len=20, unconditional_inputs=shared)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        subs = _run_engine(eng, S)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    _check_engine(m, subs, H)


@pytest.mark.skipif(not os.environ.get("PB200_FORCE_BN"), reason="run in a child process with PB200_FORCE_BN set")
def test_default_engine_weighted_child():
    from paella_b200.engine import SamplingEngine
    m, H = _default_model(), 16
    S, shared = _engine_schedule(m, H, L0=24)
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=3, max_cond_len=32, unconditional_inputs=shared)
    _check_engine(m, _run_engine(eng, S), H)


def test_default_engine_weighted_with_one_tile_width():
    _child("test_default_engine_weighted_child", {"PB200_FORCE_BN": "128"})


# ------------------------------------------------------------------ validation
def test_validation_raises_before_any_generator_moves(tiny):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    m, H, B, L = tiny[0], 8, 2, 5
    cond = _inputs(m, B, L, True, False, seed=1)
    S = m.conditioning_seq_len(cond)
    n_max = m.max_attn_weights((H, H), S)
    bad = [
        [torch.ones(3)],                                   # one entry for two samples
        [torch.ones(3)] * 3,
        [torch.ones(3), torch.ones(3, device=DEV)],        # a CUDA tensor
        [torch.ones(3), torch.ones(1, 3)],                 # not 1-D
        [torch.ones(3), torch.tensor([1.0, float("nan")])],
        [torch.ones(3), torch.tensor([float("inf")])],
        [torch.ones(3), torch.ones(n_max + 1)],            # longer than the smallest key count
    ]
    gens = _gens([1, 2])
    offs = [g.get_offset() for g in gens]
    torch.manual_seed(0)
    default_off = torch.cuda.default_generators[torch.cuda.current_device()].get_offset()
    x = torch.zeros(B, H, H, dtype=torch.int64, device=DEV)
    for aw in bad:
        with pytest.raises(ValueError):
            U.sample_notebook(m, cond, (B, H, H), steps=2, attn_weights=aw, generator=gens)
        with pytest.raises(ValueError):
            U.sample_notebook(m, cond, (B, H, H), steps=2, attn_weights=aw)
        with pytest.raises(ValueError):
            m(x, torch.ones(B, device=DEV), **cond, attn_weights=aw)
    assert [g.get_offset() for g in gens] == offs
    assert torch.cuda.default_generators[torch.cuda.current_device()].get_offset() == default_off
    U.sample_notebook(m, cond, (B, H, H), steps=1, attn_weights=[torch.ones(n_max), None], generator=gens)   # the limit is fine

    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=2, max_cond_len=10)
    g = torch.Generator(device=DEV).manual_seed(5)
    off = g.get_offset()
    one = _row(cond, 0)
    for w in (torch.ones(3, device=DEV), torch.ones(1, 3), torch.tensor([float("nan")]), torch.ones(n_max + 1),
              torch.ones(3, dtype=torch.int32), [1.0, 2.0]):
        with pytest.raises(ValueError):
            eng.submit(one, None, generator=g, cfg=None, attn_weights=w)
    assert g.get_offset() == off and not eng.busy
