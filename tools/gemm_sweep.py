#!/usr/bin/env python
"""Split the wgmma GEMM's time into main loop and per-tile cost, on the denoiser's shapes.

For every shape the GEMM is timed at K/2, K and 2K (same tile width: the planner's choice at K, pinned through
PB200_FORCE_BN in a child process) and the times are fitted to

    t = tiles_per_SM * (n_kb * t_kb + t_tile)

where tiles_per_SM is the tile count of the busiest CTA of the persistent grid and n_kb the number of 64-deep k-blocks.
The slope t_kb is the main-loop time of one k-block of one tile, the intercept t_tile what a tile costs on top of its
k-blocks and does not overlap them: the epilogue plus pipeline fill and drain.  Every window is timed with CUDA events
over at least 0.5 s of back-to-back launches after a warm-up.  Prints one JSON line.

    python tools/gemm_sweep.py [--out FILE]
"""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (M, N, K, epilogue, rows per sample): the GEMMs of one `sample` step (bench.py --workload sample)
SHAPES = [
    (8192, 5120, 1280, "gelu", 64),      # ResBlock GEMM1, level 1/2
    (32768, 2560, 640, "gelu", 256),     # ResBlock GEMM1, level 0
    (8192, 1280, 5120, "resid", 64),     # ResBlock GEMM2
    (8192, 1280, 1280, "resid", 64),     # attention out-projection
    (8192, 3840, 1280, "f16", 64),       # QKV projection
    (2048, 1280, 5120, "resid", 16),     # ResBlock GEMM2 at the lowest resolution
]
WINDOW_S = 0.5


def _time_one(M, N, K, mode, P):
    """ms per launch of one shape (the median of 3 windows of >= WINDOW_S each)."""
    import torch
    from paella_b200 import _lib, ops
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    a = torch.randn(M, K, device=dev, generator=g).half()
    w = (torch.randn(N, K, device=dev, generator=g) / math.sqrt(K)).half()
    bias = torch.randn(N, device=dev, generator=g)
    if mode == "gelu":
        out = torch.empty(M, N, device=dev, dtype=torch.float16)
        sq = torch.zeros(M // P, N, device=dev, dtype=torch.int64)
        run = lambda: ops.gemm_f16(a, w, _lib.EPI_GELU_F16, out, bias=bias, sqsum=sq, rows_per_sample=P)
    elif mode == "resid":
        out = torch.randn(M, N, device=dev, generator=g)
        film = torch.randn(M // P, 2 * N, device=dev, generator=g) * 0.1
        run = lambda: ops.gemm_f16(a, w, _lib.EPI_RESID_F32, out, bias=bias, resid=out, rows_per_sample=P, film=film)
    else:
        out = torch.empty(M, N, device=dev, dtype=torch.float16)
        run = lambda: ops.gemm_f16(a, w, _lib.EPI_F16, out, bias=bias)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def window(n):
        e0.record()
        for _ in range(n):
            run()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    window(20)                                              # warm-up: module load, tensor-map cache
    n = max(20, int(WINDOW_S * 1e3 / max(window(20) / 20, 1e-3)))
    ts = sorted(window(n) / n for _ in range(3))
    return ts[1]


def _plan(M, N, K, sms):
    from paella_b200 import _lib
    L = _lib.lib()
    bn, two, tail = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(L.pb200_gemm_plan(M, N, K, sms, ctypes.byref(bn), ctypes.byref(two), ctypes.byref(tail)), "gemm_plan")
    return bn.value


def _fit(xs, ys):
    n = len(xs)
    mx, my = sum(xs) / n, sum(ys) / n
    sxx = sum((x - mx) ** 2 for x in xs)
    slope = sum((x - mx) * (y - my) for x, y in zip(xs, ys)) / sxx
    return slope, my - slope * mx


def _gpu_info():
    import torch
    info = {"gpu": torch.cuda.get_device_name(0), "sms": torch.cuda.get_device_properties(0).multi_processor_count}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(q[0]), float(q[1])
    except Exception as e:        # the numbers are still reported, without the card's limits
        info["power_limit_w"] = f"unavailable ({type(e).__name__})"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    ap.add_argument("--one", nargs=5, metavar=("M", "N", "K", "MODE", "P"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.one:
        M, N, K, mode, P = args.one
        print(json.dumps({"ms": _time_one(int(M), int(N), int(K), mode, int(P))}), flush=True)
        return
    import torch
    assert torch.cuda.is_available(), "gemm_sweep needs a GPU"
    info = _gpu_info()
    sms = info["sms"]
    rows = []
    for M, N, K, mode, P in SHAPES:
        bn = _plan(M, N, K, sms)
        units = math.ceil(M / 128) * math.ceil(N / bn)
        tiles_per_sm = math.ceil(units / min(units, sms))
        ks = [K // 2, K, 2 * K]
        ms = {}
        for k in ks:
            env = dict(os.environ, PB200_FORCE_BN=str(bn))
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", str(M), str(N), str(k), mode, str(P)],
                               capture_output=True, text=True, env=env, cwd=ROOT)
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                raise SystemExit(f"gemm_sweep: {M}x{N}x{k} {mode} failed")
            ms[k] = json.loads(r.stdout.strip().splitlines()[-1])["ms"]
        nkb = [k // 64 for k in ks]
        slope, icpt = _fit(nkb, [ms[k] / tiles_per_sm for k in ks])      # ms per k-block / per tile, busiest CTA
        t = ms[K]
        rows.append({
            "M": M, "N": N, "K": K, "epilogue": mode, "P": P, "block_n": bn, "tiles_per_sm": tiles_per_sm,
            "ms": {str(k): round(ms[k], 4) for k in ks},
            "tflops": round(2.0 * M * N * K / t / 1e9, 1),
            "t_kb_us": round(slope * 1e3, 4),
            "t_tile_us": round(icpt * 1e3, 3),
            # main-loop rate of the whole GPU: every SM retires one 128 x BLOCK_N x 64 k-block per t_kb
            "slope_tflops": round(2.0 * 128 * bn * 64 * min(units, sms) / (slope * 1e-3) / 1e12, 1),
            "intercept_share": round(tiles_per_sm * icpt / t, 3),
        })
        print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    line = json.dumps({"metric": "gemm_sweep", **info, "shapes": rows})
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
