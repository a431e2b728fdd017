#!/bin/bash
# compute-sanitizer over the hand-rolled mbarrier / TMA / wgmma kernels (python launched DIRECTLY under the tool, not in
# attach mode).  Small shapes only: the tools run kernels 10-100x slower.
#   bash tools/sanitize.sh <tag> [outdir]  ->  <outdir>/<tag>_memcheck.log, <tag>_racecheck.log, <tag>_synccheck.log
TAG=${1:-san}
O=${2:-/tmp/paella_sanitize}
mkdir -p $O
cat > /tmp/san_case.py <<'PY'
import os, sys, math, torch
sys.path.insert(0, os.getcwd()); sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
from paella_b200 import _lib, ops
DEV = "cuda"
g = torch.Generator(device=DEV).manual_seed(0)
# wgmma GEMMs: every tile width, GELU+sqsum, RESID (+a_scale), LN fold
for (M, N, K) in [(128, 128, 64), (300, 136, 128), (512, 256, 128)]:
    a = torch.randn(M, K, device=DEV, generator=g).half(); w = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).half()
    bias = torch.randn(N, device=DEV, generator=g)
    out = torch.zeros(M, N, device=DEV); ops.gemm_f16(a, w, _lib.EPI_F32, out, bias=bias)
    o16 = torch.zeros(M, N, device=DEV, dtype=torch.float16); sq = torch.zeros(max(1, M // 4), N, device=DEV, dtype=torch.int64)
    ops.gemm_f16(a, w, _lib.EPI_GELU_F16, o16, bias=bias, sqsum=sq, rows_per_sample=4)
    x = torch.randn(M, N, device=DEV, generator=g); ops.gemm_f16(a, w, _lib.EPI_RESID_F32, x, bias=bias, resid=x)
M, N, K, P = 2048, 1280, 640, 16          # the a_scale path
a = torch.randn(M, K, device=DEV, generator=g).half(); w = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).half()
x = torch.randn(M, N, device=DEV, generator=g); s = (1 + 0.3 * torch.randn(M // P, K, device=DEV, generator=g)).half()
ops.gemm_f16(a, w, _lib.EPI_RESID_F32, x, bias=None, resid=x, rows_per_sample=P, a_scale=s)
# attention: wgmma kernel (head_dim 80: shared slots, the last slot read; a weight table) and mma.sync kernel
import test_gpu_attention_matrix as ta
for kernel, cid in (("wgmma", "slots-above-B-hd80"), ("wgmma", "table-w_row-shared-hd80"), ("mma", "hd32-P16-S20-varlen-vec5-hd32")):
    print("attn", kernel, cid, ta._run(ta._make(next(c for c in ta._cases(kernel) if c["id"] == cid))).shape)
# codec ResBlock front (row statistics + patch kernel), partial patches
from paella_b200.vqgan import ResBlock
blk = ResBlock(192, 768).to(DEV).eval()
print("vq resblock", blk(torch.randn(1, 192, 13, 13, device=DEV, generator=g)).shape)
torch.cuda.synchronize(); print("sanitizer case 1 done")
PY
cat > /tmp/san_case2.py <<'PY'
import os, sys, math, torch
sys.path.insert(0, os.getcwd()); sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
from paella_b200 import _lib, ops
DEV = "cuda"
g = torch.Generator(device=DEV).manual_seed(0)
# sampler + RNG kernels
from helpers import load_golden
from paella_b200.modules import Paella
cfg, sd, gg = load_golden("paella_tiny.npz")
m = Paella(**cfg).to(DEV).eval(); m.load_state_dict(sd)
feats = torch.randn(2 * 2 * 64, cfg["c_out"], device=DEV, generator=g)
print("sampler", m.sample_tokens(feats, 2, 8, 8, 4.0, 0.7).shape)
# per-sample streams: odd B, and 7x7 rows per sample (4 rs = 256 on this small-grid policy) -- every sample's block is partial
f3 = torch.randn(2 * 3 * 49, cfg["c_out"], device=DEV, generator=g)
gens = [torch.Generator(device=DEV).manual_seed(s) for s in (1, 2, 3)]
print("sampler per-sample", m.sample_tokens(f3, 3, 7, 7, 4.0, 0.7, gens).shape)
# per-sample (cfg, T): the per-row mix and the per-sample 1/T, on per-sample streams and on one stream (staged 1/T columns)
cfg3, t3 = torch.tensor([4.0, 1.0, 2.5]), torch.tensor([0.7, 1.2, 0.4])
gens = [torch.Generator(device=DEV).manual_seed(s) for s in (1, 2, 3)]
print("sampler params per-sample", m.sample_tokens(f3, 3, 7, 7, cfg3, t3, gens).shape)
print("sampler params one stream", m.sample_tokens(f3, 3, 7, 7, cfg3, t3).shape)
p = torch.rand(64, 100, device=DEV, generator=g); print("multinomial", ops.multinomial(p).shape)
# one-launch per-sample RNG on an odd H*W, and the sampling engine: partial CFG pairs, slot maps, a slot reused by a request
# with a shorter conditioning sequence (slot 0 frees after 1 step and takes the third request)
x7 = torch.randint(0, 64, (3, 7, 9), device=DEV, generator=g)
gens = [torch.Generator(device=DEV).manual_seed(s) for s in (1, 2, 3)]
print("randint per-sample", ops.randint(64, (3, 7, 9), DEV, gens).shape, "add_noise per-sample",
      ops.add_noise(x7, torch.tensor([0.5, -1.0, 0.9], device=DEV), None, 64, gens)[0].shape)
from paella_b200.engine import SamplingEngine
def cond(L, ci):
    d = {"byt5": torch.randn(1, L, cfg["byt5_embd"], device=DEV, generator=g), "clip": torch.randn(1, cfg["clip_embd"], device=DEV, generator=g)}
    if ci: d["clip_image"] = torch.randn(1, cfg["clip_embd"], device=DEV, generator=g)
    return d
eng = SamplingEngine(m, latent_hw=(8, 8), max_batch=2, max_cond_len=20, unconditional_inputs={k: v * 0 for k, v in cond(4, False).items()})
eng.submit(cond(12, True), generator=torch.Generator(device=DEV).manual_seed(1), steps=1)
eng.submit(cond(5, False), generator=torch.Generator(device=DEV).manual_seed(2), steps=3, cfg=None)
eng.submit(cond(2, False), generator=torch.Generator(device=DEV).manual_seed(3), steps=2, sampling_conditional_steps=1)
print("engine", [q.result.shape for q in eng.run_until_idle()])
# per-sample attn_weights: a vector longer than the conditioning (into the self keys), None and length 1; then an engine
# whose slot 0 is reused by a request with a shorter vector, and again by one with none
cw = cond(6, True); cw = {k: v.expand(3, *v.shape[1:]).contiguous() for k, v in cw.items()}
n_max = m.max_attn_weights((8, 8), m.conditioning_seq_len(cw))
print("forward per-sample weights", m(torch.randint(0, 64, (3, 8, 8), device=DEV, generator=g), torch.rand(3, device=DEV, generator=g),
      **cw, attn_weights=[torch.rand(n_max), None, torch.rand(1)]).shape)
eng = SamplingEngine(m, latent_hw=(8, 8), max_batch=2, max_cond_len=20, unconditional_inputs={k: v * 0 for k, v in cond(4, False).items()})
eng.submit(cond(12, True), generator=torch.Generator(device=DEV).manual_seed(1), steps=1, attn_weights=torch.rand(21))
eng.submit(cond(5, False), generator=torch.Generator(device=DEV).manual_seed(2), steps=3, cfg=None, attn_weights=torch.rand(3))
eng.submit(cond(2, False), generator=torch.Generator(device=DEV).manual_seed(3), steps=1, attn_weights=torch.rand(2))
eng.submit(cond(3, False), generator=torch.Generator(device=DEV).manual_seed(4), steps=1, keep_intermediates=True)
print("engine weights", [q.result.shape for q in eng.run_until_idle()])
# region sampling: the masked add-noise on an odd H*W with a slot map, region rows and a plain (all-True) row, a t < 0 row;
# then an engine whose slot 0 is reused by a request without a region
reg = torch.rand(3, 7, 9, device=DEV, generator=g) < 0.5; reg[1] = True
src7 = torch.randint(0, 64, (3, 7, 9), device=DEV, generator=g)
t7 = torch.tensor([0.5, -1.0, 0.9], device=DEV)
pool = torch.zeros_like(x7)
ops.add_noise_per_sample(x7, t7, x7, 64, ops.philox_table([torch.Generator(device=DEV).manual_seed(s) for s in (4, 5, 6)], 63, DEV),
                         pool, slot=torch.tensor([2, 0, 1], dtype=torch.int32, device=DEV), src=src7, region=reg)
print("add_noise region", ops.add_noise(x7, t7, None, 64, [torch.Generator(device=DEV).manual_seed(s) for s in (7, 8, 9)],
                                        src=src7, region=reg)[0].shape, ops.add_noise(x7, t7, x7, 64, src=src7, region=reg)[0].shape)
eng = SamplingEngine(m, latent_hw=(8, 8), max_batch=2, max_cond_len=20, unconditional_inputs={k: v * 0 for k, v in cond(4, False).items()})
eng.submit(cond(5, False), generator=torch.Generator(device=DEV).manual_seed(1), steps=1,
           init_x=torch.randint(0, 64, (1, 8, 8)), region=torch.rand(1, 8, 8) < 0.5)
eng.submit(cond(3, False), generator=torch.Generator(device=DEV).manual_seed(2), steps=2, cfg=None,
           init_x=torch.randint(0, 64, (1, 8, 8), device=DEV), region=torch.rand(1, 8, 8) < 0.3, keep_intermediates=True)
eng.submit(cond(2, False), generator=torch.Generator(device=DEV).manual_seed(3), steps=1)
print("engine regions", [q.result.shape for q in eng.run_until_idle()])
t = torch.from_numpy
print("forward", m(t(gg["x"]).to(DEV), t(gg["r"]).to(DEV), t(gg["byt5"]).to(DEV), clip=t(gg["clip"]).to(DEV)).shape)
torch.cuda.synchronize(); print("sanitizer case 2 done")
PY
for tool in memcheck racecheck; do
  for part in "" 2; do
    timeout 420 compute-sanitizer --tool $tool --print-limit 20 python -X faulthandler /tmp/san_case$part.py > $O/${TAG}_${tool}$part.log 2>&1
    echo "$tool part ${part:-1} rc=$? $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY' $O/${TAG}_${tool}$part.log | tail -1)"
  done
done
