#!/usr/bin/env python
"""Micro-benchmark of the wgmma GEMM on the denoiser's shapes (CUDA events, L2 flushed between runs)."""
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from paella_b200 import _lib, ops  # noqa: E402

SHAPES = [  # (M, N, K, mode, P)  cfg2: B'=128
    (8192, 5120, 1280, "gelu", 64), (8192, 1280, 5120, "resid", 64), (8192, 3840, 1280, "f16", 64),
    (8192, 1280, 1280, "resid", 64), (32768, 2560, 640, "gelu", 256), (32768, 640, 2560, "resid", 256),
    (2048, 5120, 1280, "gelu", 16), (2048, 1280, 5120, "resid", 16), (16896, 2560, 1280, "f16", 132),
    (65536, 8192, 256, "f16", 1024),
]


def main():
    dev = "cuda"
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    res = []
    for M, N, K, mode, P in SHAPES:
        a = torch.randn(M, K, device=dev).half()
        w = (torch.randn(N, K, device=dev) / math.sqrt(K)).half()
        bias = torch.randn(N, device=dev)
        if mode == "gelu":
            out = torch.empty(M, N, device=dev, dtype=torch.float16)
            sq = torch.zeros(M // P, N, device=dev, dtype=torch.int64)
            run = lambda: ops.gemm_f16(a, w, _lib.EPI_GELU_F16, out, bias=bias, sqsum=sq, rows_per_sample=P)
        elif mode == "resid":
            out = torch.randn(M, N, device=dev)
            run = lambda: ops.gemm_f16(a, w, _lib.EPI_RESID_F32, out, bias=bias, resid=out, rows_per_sample=P)
        else:
            out = torch.empty(M, N, device=dev, dtype=torch.float16)
            run = lambda: ops.gemm_f16(a, w, _lib.EPI_F16, out, bias=bias)
        for _ in range(3):
            run()
        ts = []
        for _ in range(10):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        t = ts[len(ts) // 2]
        # torch reference (cuBLAS fp16) for the same contraction
        tt = []
        for _ in range(5):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            torch.matmul(a, w.t())
            e1.record()
            torch.cuda.synchronize()
            tt.append(e0.elapsed_time(e1))
        tt.sort()
        r = {"M": M, "N": N, "K": K, "mode": mode, "ms": t, "tflops": 2.0 * M * N * K / t / 1e9,
             "cublas_ms": tt[len(tt) // 2], "cublas_tflops": 2.0 * M * N * K / tt[len(tt) // 2] / 1e9}
        print(json.dumps(r), flush=True)
        res.append(r)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
