"""Batch-invariant mode (``Paella.batch_invariant``, pb200_paella_set_batch_invariant): a sample's features, logits and tokens
do not depend on the batch it runs in, on the default model, with the GEMM planner free to pick its tile widths.

  * GEMM: PB200_EPI_RESID_LN_INV_F32 at BLOCK_N 64, 128 and 256 (one child process per width: PB200_FORCE_BN is read once
    per process) gives bit-identical out, out16 and ln_stat across the widths and at any row offset of a larger M; out and
    out16 equal RESID_LN's; every element within an fp64 bound
  * forward: the default model's features of a sample alone vs inside batches of 2, 5 and 64 (32x32, 64x64, 48x48; CFG pairs
    or not; mixed conditioning lengths), torch.equal with the mode on, while the planner picks several widths; the same run
    with the mode off differs
  * end to end: sample_distributed rows and a staggered SamplingEngine load equal their batch-1 calls bit for bit
  * batched engine admission writes the cache rows and kv_len that per-request write_conditioning writes, in both modes
  * two GPUs (skipped with fewer): a shard's rows equal the single-GPU rows
  * invalid use raises before anything is enqueued
"""
import ctypes
import os
import socket
import subprocess
import sys
import tempfile

import pytest
import torch

from helpers import log_jsonl

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
EPI_RESID_LN, EPI_RESID_LN_INV = 6, 8


def _log(payload):
    log_jsonl("batch_invariant.jsonl", payload)


def _gens(seeds):
    return [torch.Generator(device=DEV).manual_seed(s) for s in seeds]


def _default_model():
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    return m.to(DEV)


@pytest.fixture(scope="module")
def default_model():
    m = _default_model()
    yield m
    m.batch_invariant = False


# ------------------------------------------------------------------ 1. GEMM epilogue, every width
M_SMALL, M_BIG, N, K, P = 64, 1000, 1000, 640, 64       # N % 32 == 8: a partial last chunk
OFF = 200                                                # row offset of the embedded problem


def _gemm_inputs():
    g = torch.Generator(device="cpu").manual_seed(5)
    a = (torch.randn(M_SMALL, K, generator=g) * 0.5).half()
    w = (torch.randn(N, K, generator=g) * 0.05).half()
    bias = torch.randn(N, generator=g) * 0.1
    resid = torch.randn(M_SMALL, N, generator=g) + 3.0                 # an offset the shift removes
    shift = resid.mean(1) + 0.01 * torch.randn(M_SMALL, generator=g)
    filler = (torch.randn(M_BIG, K, generator=g) * 0.5).half()
    filler_r = torch.randn(M_BIG, N, generator=g)
    return a, w, bias, resid, shift, filler, filler_r


def _gemm_run(mode, big):
    from paella_b200 import ops
    a, w, bias, resid, shift, filler, filler_r = [t.to(DEV) for t in _gemm_inputs()]
    off = OFF if big else 0
    M = M_BIG if big else M_SMALL
    A, R, SH = filler.clone()[:M], filler_r.clone()[:M], torch.zeros(M, device=DEV)
    A[off:off + M_SMALL], R[off:off + M_SMALL], SH[off:off + M_SMALL] = a, resid, shift
    out16 = torch.empty(M, N, dtype=torch.float16, device=DEV)
    stat = torch.zeros(M, 2, dtype=torch.int64, device=DEV)
    x = R.clone()
    ops.gemm_f16(A.contiguous(), w, mode, x, bias=bias, resid=x, out16=out16, ln_stat=stat, ln_shift=SH, rows_per_sample=P)
    sl = slice(off, off + M_SMALL)
    return x[sl].cpu(), out16[sl].cpu(), stat[sl].cpu()


def _gemm_child(path):
    """Every case at this process's width (PB200_FORCE_BN): {(mode, big): (out, out16, ln_stat)}."""
    res = {(mode, big): _gemm_run(mode, big) for mode in (EPI_RESID_LN, EPI_RESID_LN_INV) for big in (False, True)}
    torch.cuda.synchronize()
    torch.save(res, path)


def _check_fp64_bound(out, out16, stat):
    a, w, bias, resid, shift, _, _ = _gemm_inputs()
    a64, w64 = a.double(), w.double()
    acc = a64 @ w64.T
    absacc = a64.abs() @ w64.abs().T
    ref = acc + bias.double() + resid.double()
    u32 = 2.0 ** -24
    bound = 2.0 ** -18 * absacc + 8 * u32 * (acc.abs() + bias.double().abs() + resid.double().abs())
    err = (out.double() - ref).abs()
    assert bool((err <= bound).all()), f"out: worst err/bound {float((err / bound).max())}"
    # the fp16 copy is the kernel's own fp32 value minus the shift, rounded once
    xs = out.double() - shift.double()[:, None]
    assert bool(((out16.double() - xs).abs() <= 2.0 ** -11 * xs.abs() + 2.0 ** -24 + u32 * out.double().abs()).all())
    # row statistics of the shifted rows: per 32-column chunk an fp32 sum (<= 32 roundings) rounded to fixed point once
    n_chunks = (N + 31) // 32
    s_ref, q_ref = xs.sum(1), (xs * xs).sum(1)
    s_got, q_got = stat[:, 0].double() / 2 ** 20, stat[:, 1].double() / 2 ** 16
    s_bound = 40 * u32 * (xs.abs().sum(1) + out.double().abs().sum(1)) + n_chunks * 2.0 ** -20
    q_bound = 80 * u32 * (xs * xs).sum(1) + 4 * u32 * (xs.abs() * out.double().abs()).sum(1) + n_chunks * 2.0 ** -16
    assert bool(((s_got - s_ref).abs() <= s_bound).all()), float(((s_got - s_ref).abs() / s_bound).max())
    assert bool(((q_got - q_ref).abs() <= q_bound).all()), float(((q_got - q_ref).abs() / q_bound).max())
    return float((err / bound).max()), float(((s_got - s_ref).abs() / s_bound).max()), float(((q_got - q_ref).abs() / q_bound).max())


def test_inv_epilogue_is_width_and_offset_invariant_at_every_width():
    res = {}
    with tempfile.TemporaryDirectory() as d:
        for bn in (64, 128, 256):
            path = os.path.join(d, f"bn{bn}.pt")
            code = f"import sys; sys.path.insert(0, {HERE!r}); import test_gpu_batch_invariant as T; T._gemm_child({path!r})"
            p = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, PB200_FORCE_BN=str(bn)), capture_output=True,
                               text=True, timeout=900, cwd=os.path.dirname(HERE))
            assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
            res[bn] = torch.load(path)
    ref = res[64][(EPI_RESID_LN_INV, False)]
    for bn in (64, 128, 256):
        for big in (False, True):
            got = res[bn][(EPI_RESID_LN_INV, big)]
            for name, x, y in zip(("out", "out16", "ln_stat"), got, ref):
                assert torch.equal(x, y), f"BLOCK_N {bn}, embedded {big}: {name} differs from BLOCK_N 64 alone"
        # the fp32 output and its fp16 copy are RESID_LN's; only the statistic's summation differs
        plain = res[bn][(EPI_RESID_LN, False)]
        assert torch.equal(plain[0], ref[0]) and torch.equal(plain[1], ref[1])
    worst = _check_fp64_bound(*ref)
    # the default epilogue's statistic does depend on the width (the reason for the INV mode)
    differs = any(not torch.equal(res[bn][(EPI_RESID_LN, False)][2], res[64][(EPI_RESID_LN, False)][2]) for bn in (128, 256))
    _log({"test": "inv_epilogue", "worst_err_over_bound": worst, "resid_ln_stat_differs_across_widths": differs})


# ------------------------------------------------------------------ 2. forward, default model, planner free
def _conditioning(m, B, L, seed=7):
    from paella_b200.synth import synthetic_conditioning
    return synthetic_conditioning(B, L, byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features,
                                  with_clip_image=True, seed=seed, device=DEV)


def _rows(d, idx):
    return {k: v[idx] for k, v in d.items()}


def _planned_widths(m, hw, batches):
    """The widths pb200_gemm_plan gives the ResBlock GEMM2s that feed an AttnBlock (RESID_LN), over the forward batches."""
    from paella_b200._lib import lib
    c = m._cfg
    widths = set()
    for B in batches:
        for lvl, (ch, kinds) in enumerate(zip(c["c_hidden"], c["level_config"])):
            if "A" not in kinds:
                continue
            Mr = B * ((hw // 2) >> lvl) ** 2
            bn = ctypes.c_int()
            assert lib().pb200_gemm_plan(Mr, ch, 4 * ch, 0, ctypes.byref(bn)) == 0
            widths.add(bn.value)
    return widths


def _features_worst(m, hw, cfg_pairs, N=64):
    cond, uncond = _conditioning(m, N, 16)
    x = torch.randint(0, m.num_labels, (N, hw, hw), device=DEV, generator=torch.Generator(device=DEV).manual_seed(11))
    r = torch.rand(N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(12))
    n_hw = hw * hw

    def run(sel):
        idx = torch.tensor(sel, device=DEV)
        groups = [_rows(cond, idx), _rows(uncond, idx)] if cfg_pairs else [_rows(cond, idx)]
        with torch.inference_mode():
            cache = m.prepare_conditioning(groups, (hw, hw))
            f = m.features(x[idx], r[idx], cache, cfg_pairs=cfg_pairs)
        B = len(sel)
        return [(f[p * n_hw:(p + 1) * n_hw], f[(B + p) * n_hw:(B + p + 1) * n_hw] if cfg_pairs else None) for p in range(B)]

    alone, worst, n_diff = {}, 0.0, 0
    for sel in ([1, 0], [3, 0, 4, 1, 2], list(range(N - 1, -1, -1))):
        got = run(sel)
        for p in (range(len(sel)) if len(sel) <= 5 else [0, 1, 30, 62, 63]):
            s = sel[p]
            if s not in alone:
                alone[s] = run([s])[0]
            for a, b in zip(got[p], alone[s]):
                if a is not None:
                    worst = max(worst, float((a - b).abs().max()))
                    n_diff += int(not torch.equal(a, b))
    per = 2 if cfg_pairs else 1
    return worst, n_diff, _planned_widths(m, hw, [per * b for b in (1, 2, 5, N)])


@pytest.mark.parametrize("cfg_pairs", [True, False], ids=["cfg", "nocfg"])
@pytest.mark.parametrize("hw", [32, 64, 48])
def test_default_forward_features_are_batch_invariant_with_the_mode_on(hw, cfg_pairs, default_model):
    assert not os.environ.get("PB200_FORCE_BN"), "this test is about the planner's own widths"
    m = default_model
    m.batch_invariant = True
    worst, n_diff, widths = _features_worst(m, hw, cfg_pairs)
    off = None
    if hw == 32 and cfg_pairs:       # the same run in the default mode is batch-dependent: the check above is not vacuous
        m.batch_invariant = False
        off = _features_worst(m, hw, cfg_pairs)[:2]
        m.batch_invariant = True
    _log({"test": "forward_batch_invariant", "hw": hw, "cfg_pairs": cfg_pairs, "widths": sorted(widths), "mode_on_max_diff": worst,
          "mode_off_max_diff": off[0] if off else None})
    assert len(widths) >= 2, f"the planner picks only {widths} over these batches"
    assert worst == 0.0 and n_diff == 0, f"mode on: {n_diff} sample blocks differ, max |diff| {worst}"
    if off is not None:
        assert off[1] > 0, "mode off: expected batch-dependent features on the default model"


# ------------------------------------------------------------------ 3. end to end
def test_default_sample_distributed_rows_equal_batch1_calls(default_model):
    from paella_b200 import utils as U
    m = default_model
    m.batch_invariant = True
    B, H = 16, 32
    seeds = list(range(300, 300 + B))
    cond, uncond = _conditioning(m, B, 12, seed=9)
    cond.pop("clip_image")
    kw = dict(steps=3, renoise_steps=2, temperature=(1.0, 0.3), cfg=(6.0, 6.0))
    gens = _gens(seeds)
    with torch.inference_mode():
        got = U.sample_distributed(m, cond, uncond, (B, H, H), generator=gens, **kw)
        for i in range(B):
            g1 = _gens([seeds[i]])
            want = U.sample_distributed(m, _rows(cond, slice(i, i + 1)), _rows(uncond, slice(i, i + 1)), (1, H, H), generator=g1, **kw)
            assert torch.equal(got[i:i + 1], want), f"row {i}"
            assert gens[i].get_offset() == g1[0].get_offset()


def _inputs(m, L, seed, zeros=False, clip=True):
    g = torch.Generator().manual_seed(seed)
    d = {"byt5": torch.randn(1, L, m.byt5_mapper.in_features, generator=g)}
    if clip:
        d["clip"] = torch.randn(1, m.clip_mapper.in_features, generator=g)
    return {k: (torch.zeros_like(v) if zeros else v).to(DEV) for k, v in d.items()}


def test_default_staggered_engine_requests_equal_batch1_calls(default_model):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    from paella_b200.vqgan import VQModel
    m = default_model
    m.batch_invariant = True
    H = W = 32
    torch.manual_seed(0)
    vq = VQModel(levels=2, bottleneck_blocks=1, c_hidden=32, c_latent=4, codebook_size=m.num_labels).to(DEV)
    g = torch.Generator().manual_seed(50)
    region = torch.rand(1, H, W, generator=g) < 0.5
    init_x = torch.randint(0, m.num_labels, (1, H, W), generator=g)
    S = {0: [dict(seed=1, steps=3, L=12), dict(seed=2, steps=2, L=7, cfg=None), dict(seed=3, steps=4, L=12),
             dict(seed=4, steps=3, L=12, attn_weights=torch.linspace(0.5, 1.5, 6))],
         1: [dict(seed=5, steps=2, L=5, mode="argmax"), dict(seed=6, steps=3, L=12, init_x=init_x, region=region)],
         2: [dict(seed=7, steps=3, L=9, mode="quant", cfg=(4.0, 2.0)), dict(seed=8, steps=1, L=12)],
         3: [dict(seed=9, steps=4, L=12, sampling_quant_steps=2, own_uncond=True)]}
    keys = ("steps", "cfg", "init_x", "region", "mode", "sampling_quant_steps", "attn_weights")
    shared = _inputs(m, 4, 0, zeros=True)
    eng = SamplingEngine(m, latent_hw=(H, W), max_batch=6, max_cond_len=20, unconditional_inputs=shared, vqmodel=vq)
    subs, step = [], 0
    with torch.inference_mode():
        while step <= max(S) or eng.busy:
            for sp in S.get(step, []):
                sp["inputs"] = _inputs(m, sp["L"], 100 + sp["seed"])
                sp["uncond"] = _inputs(m, 3, 0, zeros=True, clip=False) if sp.get("own_uncond") else shared
                kw = {k: sp[k] for k in keys if k in sp}
                gen = torch.Generator(device=DEV).manual_seed(sp["seed"])
                subs.append((sp, eng.submit(sp["inputs"], sp["uncond"] if sp.get("own_uncond") else None, generator=gen,
                                            keep_intermediates=True, **kw), gen))
            eng.step()
            step += 1
        for sp, req, gen in subs:
            kw = {k: sp[k] for k in keys if k in sp}
            g1 = torch.Generator(device=DEV).manual_seed(sp["seed"])
            want, inter = U.sample_notebook(m, sp["inputs"], (1, H, W), sp["uncond"], vqmodel=vq, generator=[g1], **kw)
            assert torch.equal(req.result, want), sp
            assert len(req.intermediates) == len(inter) and all(torch.equal(a, b) for a, b in zip(req.intermediates, inter)), sp
            assert gen.get_offset() == g1.get_offset(), sp


# ------------------------------------------------------------------ 4. batched admission
@pytest.mark.parametrize("mode_on", [False, True], ids=["default", "batch_invariant"])
def test_batched_admission_writes_what_per_request_writes(mode_on, default_model):
    from paella_b200.engine import SamplingEngine
    from paella_b200.modules import ConditioningCache
    m = default_model
    m.batch_invariant = mode_on
    H = W = 16
    shared = _inputs(m, 4, 0, zeros=True)
    eng = SamplingEngine(m, latent_hw=(H, W), max_batch=6, max_cond_len=16, unconditional_inputs=shared)
    ref = ConditioningCache(torch.zeros_like(eng.cache.cache), eng.n_slots, eng.s_max, eng.n_slots, None)
    with torch.inference_mode():
        m.write_conditioning(ref, eng.shared_slot, shared, (H, W))

        def admit(specs):
            reqs = []
            for sp in specs:
                inputs = _inputs(m, sp["L"], sp["seed"], clip=sp.get("clip", True))
                unc = _inputs(m, sp["uL"], sp["seed"] + 1, clip=False) if sp.get("uL") else None
                g = torch.Generator(device=DEV).manual_seed(sp["seed"])
                reqs.append((eng.submit(inputs, unc, generator=g, steps=sp["steps"], cfg=(3.0, 3.0)), inputs, unc))
            eng.step()
            for req, inputs, unc in reqs:            # the per-request writes, at the slots the engine chose
                m.write_conditioning(ref, req.slot, inputs, (H, W))
                if unc is not None:
                    m.write_conditioning(ref, req.uncond_slot, unc, (H, W))
            return reqs

        # one layout, own unconditional rows for some (slots 0-3, 6, 7, 9)
        first = admit([dict(L=10, seed=1, steps=1, uL=5), dict(L=10, seed=2, steps=3, uL=5), dict(L=10, seed=3, steps=1),
                       dict(L=10, seed=4, steps=3, uL=5)])
        assert torch.equal(eng.cache.cache, ref.cache)
        assert [r.slot for r, _, _ in first] == [0, 1, 2, 3]
        # slots 0 and 2 retired: the next admission gets non-contiguous free slots, mixed layouts and both kinds of uncond
        second = admit([dict(L=10, seed=5, steps=2), dict(L=7, seed=6, steps=2, clip=False, uL=7), dict(L=7, seed=7, steps=2, clip=False, uL=7),
                        dict(L=12, seed=8, steps=2, uL=5)])
        assert [r.slot for r, _, _ in second] == [0, 2, 4, 5]
        assert torch.equal(eng.cache.cache, ref.cache)
        eng.run_until_idle()


# ------------------------------------------------------------------ 5. two GPUs
TOTAL2, H2, SEEDS2 = 6, 16, [70, 71, 72, 73, 74, 75]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _two_gpu_inputs(m):
    from paella_b200.synth import synthetic_conditioning
    return synthetic_conditioning(TOTAL2, 8, seed=7, byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features)


def _worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    sys.path.insert(0, HERE)
    from paella_b200 import parallel as P
    from paella_b200 import utils as U
    m = _default_model().to(dev)
    m.batch_invariant = True
    cond, uncond = _two_gpu_inputs(m)
    lo, hi = P.shard_range(TOTAL2, rank, world)
    gens = [torch.Generator(device=dev).manual_seed(s) for s in SEEDS2[lo:hi]]
    with torch.inference_mode():
        toks = U.sample(m, {k: v[lo:hi].to(dev) for k, v in cond.items()}, (hi - lo, H2, H2),
                        {k: v[lo:hi].to(dev) for k, v in uncond.items()}, steps=3, renoise_steps=2, generator=gens)
    full = P.gather_tokens(toks, [P.shard_range(TOTAL2, r, world)[1] - P.shard_range(TOTAL2, r, world)[0] for r in range(world)])
    if rank == 0:
        ret["full"] = full.cpu()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_shards_equal_single_gpu_rows_with_the_mode_on(default_model):
    import torch.multiprocessing as mp
    from paella_b200 import utils as U
    m = default_model
    m.batch_invariant = True
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    cond, uncond = _two_gpu_inputs(m)
    with torch.inference_mode():
        want = U.sample(m, {k: v.to(DEV) for k, v in cond.items()}, (TOTAL2, H2, H2), {k: v.to(DEV) for k, v in uncond.items()},
                        steps=3, renoise_steps=2, generator=_gens(SEEDS2))
    assert torch.equal(ret["full"], want.cpu())


# ------------------------------------------------------------------ 6. invalid use
def test_invalid_use_raises_before_anything_is_enqueued():
    from helpers import load_golden
    from paella_b200 import _lib, ops
    from paella_b200._lib import PaellaB200Error, lib
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).eval()
    m.load_state_dict(sd)
    # no handle yet: the value is kept and applied when the weights are packed
    assert m._handle is None and m.batch_invariant is False
    m.batch_invariant = True
    assert m.batch_invariant is True and m._handle is None
    for bad in (1, "yes", None, 1.0):
        with pytest.raises(TypeError):
            m.batch_invariant = bad
    assert m.batch_invariant is True
    m = m.to(DEV)
    m._ensure_packed()
    n0 = lib().pb200_launch_count()
    with pytest.raises(TypeError):
        m.batch_invariant = 0
    assert m.batch_invariant is True
    m.batch_invariant = False
    # the C entry point: null handle, out-of-range value
    assert lib().pb200_paella_set_batch_invariant(None, 1) != 0
    assert lib().pb200_paella_set_batch_invariant(m._handle, 2) != 0
    assert lib().pb200_paella_set_batch_invariant(m._handle, -1) != 0
    assert lib().pb200_launch_count() == n0
    # the epilogue's own requirements, checked before the launch
    a = torch.zeros(128, 64, dtype=torch.float16, device=DEV)
    w = torch.zeros(64, 64, dtype=torch.float16, device=DEV)
    x = torch.zeros(128, 64, device=DEV)
    with pytest.raises(PaellaB200Error, match="RESID_LN needs out16"):
        ops.gemm_f16(a, w, _lib.EPI_RESID_LN_INV_F32, x, resid=x)
    with pytest.raises(PaellaB200Error, match="without resid"):
        ops.gemm_f16(a, w, _lib.EPI_RESID_LN_INV_F32, x, out16=x.half(), ln_stat=torch.zeros(128, 2, dtype=torch.int64, device=DEV))
    assert lib().pb200_launch_count() == n0
