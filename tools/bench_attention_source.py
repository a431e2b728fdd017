"""Prompt-to-prompt editing, timed in one process with the arms alternating, on the default model with CFG 8, temperature
(1.0, 0.2), 8 steps, L_byt5=128+clip and per-sample generators, at bench.py's ``sample`` shape (bs 64, 32x32 latents):

  * plain: ``sample()`` on 64 samples without attention_source;
  * edit_k8: 32 sources and 32 edits (edit 32 + i replays source i, on its own prompt and the source's seed), k = steps;
  * edit_k4: the same with k = steps / 2;
  * engine_plain / engine_edit: a SamplingEngine (max_batch 64) serving 256 requests queued at once, without edits and with half
    of them edits of the other half (each source submitted right before its edit).

An edit row loads its source's Q and K instead of its own, so the attention kernels read the same bytes; the arms differ only in
which kernel instance runs and in where the K loads point.  A second, profiled run of the sample() arms (torch.profiler, separate
from the timed rounds) sums the device time of the attention kernels.

  python tools/bench_attention_source.py [--rounds 3]

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
    from paella_b200.engine import SamplingEngine
    from paella_b200.synth import synthetic_conditioning
    from torch.profiler import ProfilerActivity, profile
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    model = bench.build_model(dev)
    model.pack_weights()
    STEPS, B, H, N_ENG = 8, 64, 32, 256
    kw = dict(temperature=(1.0, 0.2), steps=STEPS, renoise_steps=STEPS - 1, cfg=8.0)
    cond, uncond = synthetic_conditioning(B, bench.BYT5_LEN, seed=1234, device=dev)
    half = B // 2
    sources = {"plain": None,
               "edit_k8": [None] * half + [(i, STEPS) for i in range(half)],
               "edit_k4": [None] * half + [(i, STEPS // 2) for i in range(half)]}
    seeds = list(range(half)) * 2                      # edit 32 + i shares source i's seed

    def gens(seed_list):
        return [torch.Generator(device=dev).manual_seed(s) for s in seed_list]

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    def run_sample(arm):
        return lambda: U.sample(model, cond, (B, H, H), uncond, generator=gens(seeds), attention_source=sources[arm], **kw)

    row = lambda d, i: {k: v[i:i + 1] for k, v in d.items()}          # noqa: E731
    eng = SamplingEngine(model, latent_hw=(H, H), max_batch=B, max_cond_len=bench.BYT5_LEN + 4, unconditional_inputs=row(uncond, 0))

    def run_engine(arm):
        def f():
            g = gens([i // 2 for i in range(N_ENG)])
            for i in range(0, N_ENG, 2):
                src = eng.submit(row(cond, i % B), generator=g[i], steps=STEPS, renoise_steps=STEPS - 1, cfg=(8.0, 8.0),
                                 temperature=(1.0, 0.2))
                eng.submit(row(cond, (i + 1) % B), generator=g[i + 1], steps=STEPS, renoise_steps=STEPS - 1, cfg=(8.0, 8.0),
                           temperature=(1.0, 0.2), attention_source=(src, STEPS) if arm == "engine_edit" else None)
            eng.run_until_idle()
        return f

    arms = {"plain": (run_sample, B), "edit_k8": (run_sample, B), "edit_k4": (run_sample, B),
            "engine_plain": (run_engine, N_ENG), "engine_edit": (run_engine, N_ENG)}
    for a, (mk, _) in arms.items():                    # warm-up: every shape the timed windows use
        mk(a)()
    rates = {a: [] for a in arms}
    for _ in range(args.rounds):
        for a, (mk, n) in arms.items():
            rates[a].append(n / timed(mk(a)))
    prof_ms = {}
    for a in ("plain", "edit_k8"):                     # a profiled run of its own per arm
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run_sample(a)()
            torch.cuda.synchronize()
        prof_ms[a] = sum(e.device_time_total for e in prof.key_averages() if "attention" in e.key) / 1e3
    med = {k: statistics.median(v) for k, v in rates.items()}
    res = {"gpu": gpu_info(), "rounds": args.rounds, "steps": STEPS, "batch": B, "latent": H, "engine_requests": N_ENG,
           "images_per_s": rates, "median_images_per_s": med, "range_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
           "edit_k8_over_plain": med["edit_k8"] / med["plain"], "edit_k4_over_plain": med["edit_k4"] / med["plain"],
           "engine_edit_over_plain": med["engine_edit"] / med["engine_plain"], "profiled_attention_device_ms_per_call": prof_ms}
    for k in arms:
        print(f"[bench_attention_source] {k}: {med[k]:.2f} img/s ({min(rates[k]):.2f}-{max(rates[k]):.2f})", file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
