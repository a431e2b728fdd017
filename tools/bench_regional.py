"""Regional prompts, timed in one process with the arms alternating (default model, 32x32 latents, L_byt5=128+clip, CFG 8,
temperature (1.0, 0.2), 8 steps):

  * sample: ``sample()`` at bs 64 with per-sample generators (the shape of bench.py's ``sample`` workload), plain, with 2 regions
    per sample (left and right halves) and with 4 (the quadrants); every region prompt has the base prompt's layout;
  * engine: 256 requests through SamplingEngine, max_batch 64 (tools/bench_engine.py's uniform load), plain on an engine built
    without regional slots and with 2 regions per request on one built with max_prompt_regions=2.

Then one profiled call per arm gives the device time of the attention kernels and of the regional_masks kernel.

  python tools/bench_regional.py [--rounds 3]

Prints one JSON line with every round, medians and ranges, the kernel-family times, and the GPU name, power limit and maximum SM
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


def halves(H):
    left = torch.zeros(H, H, dtype=torch.bool)
    left[:, :H // 2] = True
    return [left, ~left]


def quadrants(H):
    out = []
    for y in (0, 1):
        for x in (0, 1):
            q = torch.zeros(H, H, dtype=torch.bool)
            q[y * H // 2:(y + 1) * H // 2, x * H // 2:(x + 1) * H // 2] = True
            out.append(q)
    return out


def main():
    import bench
    from bench_per_sample_params import gpu_info
    from torch.profiler import ProfilerActivity, profile
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
    H, B, N, STEPS = 32, 64, 256, 8
    cond, uncond = synthetic_conditioning(B, bench.BYT5_LEN, seed=1234, device=dev)
    extra, _ = synthetic_conditioning(4 * B, bench.BYT5_LEN, seed=4321, device=dev)
    row = lambda d, i: {k: v[i:i + 1] for k, v in d.items()}          # noqa: E731
    kw = dict(temperature=(1.0, 0.2), steps=STEPS, renoise_steps=STEPS - 1)
    layouts = {"plain": [], "2 regions": halves(H), "4 regions": quadrants(H)}

    def regions(name, b):
        return [(row(extra, 4 * b + k), reg) for k, reg in enumerate(layouts[name])] or None

    per_sample = {a: [regions(a, b) for b in range(B)] if layouts[a] else None for a in layouts}
    per_request = {a: [regions(a, i % B) for i in range(N)] for a in ("plain", "2 regions")}
    engines = {"plain": SamplingEngine(model, latent_hw=(H, H), max_batch=B, max_cond_len=bench.BYT5_LEN + 4,
                                       unconditional_inputs=row(uncond, 0)),
               "2 regions": SamplingEngine(model, latent_hw=(H, H), max_batch=B, max_cond_len=bench.BYT5_LEN + 4,
                                           unconditional_inputs=row(uncond, 0), max_prompt_regions=2)}

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
        return lambda: U.sample(model, cond, (B, H, H), uncond, cfg=8.0, generator=gens(B, 0), prompt_regions=per_sample[a], **kw)

    def engine_run(a):
        def f():
            g, eng = gens(N, 0), engines[a]
            for i in range(N):
                eng.submit(row(cond, i % B), generator=g[i], cfg=(8.0, 8.0), prompt_regions=per_request[a][i], **kw)
            eng.run_until_idle()
        return f

    arms = [("sample", a, sample_run(a), B) for a in layouts] + [("engine", a, engine_run(a), N) for a in engines]
    rates = {f"{ld}/{a}": [] for ld, a, _, _ in arms}
    for _, _, f, _ in arms:                    # warm-up: every shape the timed windows use
        f()
    for _ in range(args.rounds):
        for ld, a, f, n in arms:
            rates[f"{ld}/{a}"].append(n / timed(f))
    families = {}
    for ld, a, f, _ in arms:                   # profiled separately: tracing slows the host
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            f()
            torch.cuda.synchronize()
        ms = {"attention": 0.0, "regional_masks": 0.0}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                fam = "regional_masks" if "regional_masks" in e.name else "attention" if "attention" in e.name else None
                if fam:
                    ms[fam] += e.device_time_total / 1e3
        families[f"{ld}/{a}"] = ms
    med = {k: statistics.median(v) for k, v in rates.items()}
    res = {"gpu": gpu_info(), "rounds": args.rounds, "batch": B, "latent": H, "steps": STEPS, "engine_requests": N,
           "images_per_s": rates, "median_images_per_s": med, "range_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
           "kernel_ms_per_call": families}
    for k in rates:
        print(f"[bench_regional] {k}: {med[k]:.2f} img/s ({min(rates[k]):.2f}-{max(rates[k]):.2f}); attention "
              f"{families[k]['attention']:.1f} ms, regional_masks {families[k]['regional_masks']:.2f} ms", file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
