"""Cost of region sampling (inpainting / outpainting), timed in one process with the arms alternating so that all see the same
clocks and neighbours.  The `sample` workload's shape of bench.py (default model, bs 64, 32x32 latents, L_byt5=128+clip,
CFG 8, temperature (1.0, 0.2), 8 steps):

  * `plain`: sample_distributed without init_x or region;
  * `region`: the same call inpainting the right half of every image (init_x + region);
  * `engine_plain` / `engine_half_region`: 256 requests of 8 steps through SamplingEngine (max_batch 64), none or every second
    one inpainting the right half.

  python tools/bench_inpaint.py [--rounds 3]

Prints one JSON line: images/s per arm and round, the medians, and the GPU name and power limit read in the same run.
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
    w = bench.WORKLOADS["sample"]
    B, H, steps, L = w["batch"], w["latent"], w["steps"], bench.BYT5_LEN
    cond, uncond = synthetic_conditioning(B, L, seed=1234, device=dev)
    kw = dict(steps=steps, renoise_steps=steps - 1, temperature=(1.0, 0.2), cfg=(8.0, 8.0))
    init_x = torch.randint(0, model.num_labels, (B, H, H), generator=torch.Generator().manual_seed(5)).to(dev)
    region = torch.zeros(B, H, H, dtype=torch.bool)
    region[:, :, H // 2:] = True
    row = lambda d, i: {k: v[i:i + 1] for k, v in d.items()}          # noqa: E731
    N = 256
    eng = SamplingEngine(model, latent_hw=(H, H), max_batch=B, max_cond_len=L + 4, unconditional_inputs=row(uncond, 0))

    def engine_run(with_region):
        g = [torch.Generator(device=dev).manual_seed(i) for i in range(N)]
        for i in range(N):
            extra = dict(init_x=init_x[i % B:i % B + 1], region=region[i % B:i % B + 1]) if with_region and i % 2 else {}
            eng.submit(row(cond, i % B), generator=g[i], **kw, **extra)
        eng.run_until_idle()

    arms = {
        "plain": lambda: U.sample_distributed(model, cond, uncond, (B, H, H), **kw),
        "region": lambda: U.sample_distributed(model, cond, uncond, (B, H, H), init_x=init_x, region=region, **kw),
        "engine_plain": lambda: engine_run(False),
        "engine_half_region": lambda: engine_run(True),
    }
    n_img = {k: (N if k.startswith("engine") else B) for k in arms}
    for f in arms.values():           # warm-up: every shape the timed windows use
        f()
    torch.cuda.synchronize()
    rates = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, f in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            rates[k].append(n_img[k] / (e0.elapsed_time(e1) / 1e3))
    med = {k: statistics.median(v) for k, v in rates.items()}
    res = {"gpu": gpu_info(), "rounds": args.rounds, "batch": B, "latent": H, "steps": steps, "byt5_len": L,
           "engine_requests": N, "images_per_s": rates, "median_images_per_s": med,
           "spread_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
           "region_vs_plain": med["region"] / med["plain"],
           "engine_half_region_vs_plain": med["engine_half_region"] / med["engine_plain"]}
    for k in arms:
        print(f"[bench_inpaint] {k}: {med[k]:.2f} img/s (rounds {', '.join(f'{r:.2f}' for r in rates[k])})",
              file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
