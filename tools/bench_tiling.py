"""Seamless tiling, timed in one process with the plain and 'xy' arms alternating (default model, 32x32 latents, L_byt5=128+clip,
CFG 8, temperature (1.0, 0.2), 8 steps; the default-size f4 codec):

  * sample: ``sample()`` at bs 64 with per-sample generators (the shape of bench.py's ``sample`` workload);
  * engine: 256 requests through SamplingEngine, max_batch 64 (tools/bench_engine.py's uniform load);
  * decode: ``decode_indices_u8`` of 256 token grids of 64x64 (256x256 images).

  python tools/bench_tiling.py [--rounds 3]

Prints one JSON line with every round, medians and ranges, and the GPU name, power limit and maximum SM clock of the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    import bench
    from bench_per_sample_params import gpu_info
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    from paella_b200.synth import synthetic_conditioning
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    model = bench.build_model(dev)
    model.pack_weights()
    vq = bench.build_vqgan(dev)
    H, B, N, STEPS, NDEC = 32, 64, 256, 8, 256
    cond, uncond = synthetic_conditioning(B, bench.BYT5_LEN, seed=1234, device=dev)
    row = lambda d, i: {k: v[i:i + 1] for k, v in d.items()}          # noqa: E731
    kw = dict(temperature=(1.0, 0.2), steps=STEPS, renoise_steps=STEPS - 1)
    arms = {"plain": None, "xy": "xy"}
    eng = SamplingEngine(model, latent_hw=(H, H), max_batch=B, max_cond_len=bench.BYT5_LEN + 4, unconditional_inputs=row(uncond, 0))
    toks = torch.randint(0, 8192, (NDEC, 64, 64), generator=torch.Generator().manual_seed(3)).to(dev)

    def gens(n, base):
        return [torch.Generator(device=dev).manual_seed(base + i) for i in range(n)]

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    def sample_run(a):
        return lambda: U.sample(model, cond, (B, H, H), uncond, cfg=8.0, generator=gens(B, 0), tiling=arms[a], **kw)

    def engine_run(a):
        def f():
            g = gens(N, 0)
            for i in range(N):
                eng.submit(row(cond, i % B), generator=g[i], cfg=(8.0, 8.0), tiling=arms[a], **kw)
            eng.run_until_idle()
        return f

    def decode_run(a):
        return lambda: vq.decode_indices_u8(toks, arms[a])

    loads = {"sample": (sample_run, B), "engine": (engine_run, N), "decode": (decode_run, NDEC)}
    rates = {f"{ld}/{a}": [] for ld in loads for a in arms}
    for ld, (mk, _) in loads.items():          # warm-up: every shape the timed windows use
        for a in arms:
            mk(a)()
    for _ in range(args.rounds):
        for ld, (mk, n) in loads.items():
            for a in arms:
                rates[f"{ld}/{a}"].append(n / timed(mk(a)))
    med = {k: statistics.median(v) for k, v in rates.items()}
    res = {"gpu": gpu_info(), "rounds": args.rounds, "batch": B, "latent": H, "steps": STEPS, "engine_requests": N,
           "decode_images": NDEC, "images_per_s": rates, "median_images_per_s": med,
           "range_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()}}
    for k in rates:
        print(f"[bench_tiling] {k}: {med[k]:.2f} img/s ({min(rates[k]):.2f}-{max(rates[k]):.2f})", file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
