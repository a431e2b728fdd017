"""Attention maps, timed in one process with the arms alternating: ``sample()`` on the default model with CFG 8, temperature
(1.0, 0.2), 8 steps, L_byt5=128+clip and per-sample generators, at the shapes of bench.py's ``sample`` (bs 64, 32x32 latents) and
``sample64`` (bs 16, 64x64) workloads:

  * plain: attention_maps=False;
  * maps: attention_maps=True (every sample's maps).

The maps arm runs the maps instance of the attention kernel, which also writes each conditioning score and each query's
log-sum-exp to a workspace, then an accumulate kernel per AttnBlock that reads them back, and one finalize kernel per call.  A
second, profiled run of each arm (torch.profiler, separate from the timed rounds) sums the device time of the attention family:
the attention kernels and the two map kernels, listed on their own.

  python tools/bench_attention_maps.py [--rounds 3]

Prints one JSON line with every round, medians and ranges, the profiled kernel times, and the GPU name, power limit and maximum SM
clock of the same run.
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
    from paella_b200.synth import synthetic_conditioning
    from torch.profiler import ProfilerActivity, profile
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    model = bench.build_model(dev)
    model.pack_weights()
    STEPS = 8
    shapes = {"bs64_32x32": (64, 32), "bs16_64x64": (16, 64)}
    arms = ("plain", "maps")
    kw = dict(temperature=(1.0, 0.2), steps=STEPS, renoise_steps=STEPS - 1, cfg=8.0)

    def gens(n, base):
        return [torch.Generator(device=dev).manual_seed(base + i) for i in range(n)]

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    res = {"gpu": gpu_info(), "rounds": args.rounds, "steps": STEPS, "shapes": {}}
    for name, (B, H) in shapes.items():
        cond, uncond = synthetic_conditioning(B, bench.BYT5_LEN, seed=1234, device=dev)

        def run(arm):
            return lambda: U.sample(model, cond, (B, H, H), uncond, generator=gens(B, 0), attention_maps=arm == "maps", **kw)
        rates = {a: [] for a in arms}
        for a in arms:                         # warm-up: every shape the timed windows use
            run(a)()
        for _ in range(args.rounds):
            for a in arms:
                rates[a].append(B / timed(run(a)))
        prof_ms = {}
        for a in arms:                         # a profiled run of its own per arm
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run(a)()
                torch.cuda.synchronize()
            fam = {"attention": 0.0, "attention_maps_accumulate": 0.0, "attention_maps_finalize": 0.0}
            for e in prof.key_averages():
                if "attention_maps_accumulate" in e.key:
                    fam["attention_maps_accumulate"] += e.device_time_total / 1e3
                elif "attention_maps_finalize" in e.key:
                    fam["attention_maps_finalize"] += e.device_time_total / 1e3
                elif "attention" in e.key:
                    fam["attention"] += e.device_time_total / 1e3
            prof_ms[a] = fam
        med = {k: statistics.median(v) for k, v in rates.items()}
        res["shapes"][name] = {"batch": B, "latent": H, "images_per_s": rates, "median_images_per_s": med,
                               "range_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
                               "maps_over_plain": med["maps"] / med["plain"], "profiled_device_ms_per_call": prof_ms}
        for k in arms:
            print(f"[bench_attention_maps] {name} {k}: {med[k]:.2f} img/s ({min(rates[k]):.2f}-{max(rates[k]):.2f}); "
                  f"profiled ms {json.dumps({f: round(v, 2) for f, v in prof_ms[k].items()})}", file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
