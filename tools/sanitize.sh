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
# attention: wgmma kernel (head_dim 80) and mma.sync kernel
import test_gpu_attention as ta
print("attn wgmma", ta._run(2, 64, 20, 2, 80, True, True, False)[:2])
print("attn wgmma P=16", ta._run(2, 16, 12, 2, 80, True, False, True)[:2])
print("attn mma", ta._run(2, 16, 12, 2, 32, True, True, False)[:2])
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
p = torch.rand(64, 100, device=DEV, generator=g); print("multinomial", ops.multinomial(p).shape)
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
