"""Confidence-guided renoising, timed in one process with the arms alternating over the rounds:

  * ``sample()`` on the default model at bs 64, 32x32 latents, L_byt5=128+clip, CFG 8, 8 steps, per-sample generators (bench.py's
    ``sample`` shape), and at bs 16, 64x64 latents, 12 steps (bench.py's ``sample64`` shape, without its CLIP-image conditioning),
    each in four arms: plain, every sample at tau = 0, every sample at tau = 2, and half the batch at tau = 2;
  * the engine's uniform load: 256 requests of 8 steps queued at once on an engine with max_batch = 64 at 32x32, plain and with
    every request at tau = 2.

A renoising step then adds one out_mapper GEMM with its log-sum-exp (token_logprob_kernel) and replaces the add-noise launch by the
selection (renoise_confidence_kernel).  A separate torch.profiler pass over one call of each workload gives the device time of the
two new kernels per call.

  python tools/bench_confidence.py [--rounds 3]

Prints one JSON line with every round, medians and ranges, the kernel times, and the GPU name, power limit and maximum SM clock of
the same run.
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

    def gens(n, base):
        return [torch.Generator(device=dev).manual_seed(base + i) for i in range(n)]

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    shapes = {"sample": (64, 32, 8), "sample64": (16, 64, 12)}
    arms = {}
    for name, (B, H, steps) in shapes.items():
        cond, uncond = synthetic_conditioning(B, bench.BYT5_LEN, seed=1234, device=dev)
        kw = dict(temperature=(1.0, 0.2), steps=steps, renoise_steps=steps - 1, cfg=8.0)
        for arm, conf in (("plain", None), ("tau0", 0.0), ("tau2", 2.0), ("half", [2.0 if b % 2 else None for b in range(B)])):
            arms[f"{name}/{arm}"] = (B, lambda cond=cond, uncond=uncond, B=B, H=H, kw=kw, conf=conf:
                                     U.sample(model, cond, (B, H, H), uncond, generator=gens(B, 0), confidence_renoise=conf, **kw))
    H, MB, N = 32, 64, 256
    cond, uncond = synthetic_conditioning(MB, bench.BYT5_LEN, seed=1234, device=dev)
    row = lambda d, i: {k: v[i:i + 1] for k, v in d.items()}          # noqa: E731
    eng = SamplingEngine(model, latent_hw=(H, H), max_batch=MB, max_cond_len=bench.BYT5_LEN + 4, unconditional_inputs=row(uncond, 0))

    def engine_run(conf):
        g = gens(N, 0)
        for i in range(N):
            eng.submit(row(cond, i % MB), generator=g[i], steps=8, renoise_steps=7, cfg=(8.0, 8.0), temperature=(1.0, 0.2),
                       confidence_renoise=conf)
        eng.run_until_idle()
    for arm, conf in (("plain", None), ("tau2", 2.0)):
        arms[f"engine/{arm}"] = (N, lambda conf=conf: engine_run(conf))

    rates = {a: [] for a in arms}
    for a, (_, f) in arms.items():          # warm-up: every shape the timed windows use
        f()
    for _ in range(args.rounds):
        for a, (n, f) in arms.items():
            rates[a].append(n / timed(f))

    # device time of the two new kernels per call, in a profiler pass of its own
    from torch.profiler import ProfilerActivity, profile
    kernels = {}
    for a in ("sample/tau2", "sample64/tau2", "engine/tau2"):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            arms[a][1]()
            torch.cuda.synchronize()
        tot = {"token_logprob": 0.0, "renoise_confidence": 0.0, "all": 0.0}
        cnt = {"token_logprob": 0, "renoise_confidence": 0}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            us = e.device_time if hasattr(e, "device_time") else e.cuda_time
            tot["all"] += us
            for k in cnt:
                if k in e.name:
                    tot[k] += us
                    cnt[k] += 1
        kernels[a] = {"device_us": tot, "launches": cnt,
                      "share_of_device_time": {k: tot[k] / tot["all"] for k in cnt} if tot["all"] else None}

    med = {k: statistics.median(v) for k, v in rates.items()}
    names = list(shapes) + ["engine"]
    out = {"gpu": gpu_info(), "rounds": args.rounds, "images_per_s": rates, "median_images_per_s": med,
           "range_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
           "time_over_plain": {f"{n}/{arm}": med[f"{n}/plain"] / med[f"{n}/{arm}"] for n in names for arm in ("tau0", "tau2", "half")
                               if f"{n}/{arm}" in med},
           "kernels": kernels}
    for k in rates:
        print(f"[bench_confidence] {k}: {med[k]:.2f} img/s ({min(rates[k]):.2f}-{max(rates[k]):.2f})", file=sys.stderr, flush=True)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
