"""SamplingEngine against closed sample() batches, timed in one process with the arms alternating so that all see the same
clocks and neighbours (default model, 32x32 latents, L_byt5=128+clip, CFG 8, temperature (1.0, 0.2)):

  * uniform load: 256 requests of 8 steps submitted at once to an engine with max_batch=64, against four sample() calls of
    64 with per-sample generators -- the same work, so the rates should agree;
  * mixed load: --mixed requests with steps drawn from {8, 12, 16}, all queued at t=0 so that 64 are in flight at every step
    (a closed loop), against static batching that groups the requests by step count into sample() calls of up to 64.
    Reports images/s and the p50 / p95 request latency (queue time included; CUDA events, no host synchronisation inside
    the timed window).

  python tools/bench_engine.py [--rounds 3] [--mixed 192]

Prints one JSON line with every round, the medians and the spread, and the GPU name and power limit read in the same run.
"""
import argparse
import json
import os
import random
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
    ap.add_argument("--mixed", type=int, default=192, help="requests of the mixed load")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    model = bench.build_model(dev)
    model.pack_weights()
    H, MB, N_UNI = 32, 64, 256
    cond, uncond = synthetic_conditioning(MB, bench.BYT5_LEN, seed=1234, device=dev)
    row = lambda d, i: {k: v[i:i + 1] for k, v in d.items()}          # noqa: E731
    kw = dict(temperature=(1.0, 0.2))
    rng = random.Random(0)
    mixed_steps = [rng.choice([8, 12, 16]) for _ in range(args.mixed)]
    eng = SamplingEngine(model, latent_hw=(H, H), max_batch=MB, max_cond_len=bench.BYT5_LEN + 4,
                         unconditional_inputs=row(uncond, 0))

    def gens(n, base):
        return [torch.Generator(device=dev).manual_seed(base + i) for i in range(n)]

    def engine_run(steps_list):
        """-> (seconds, [latency ms]): every request queued at t=0."""
        start = torch.cuda.Event(enable_timing=True)
        start.record()
        g = gens(len(steps_list), 0)
        reqs = [eng.submit(row(cond, i % MB), generator=g[i], steps=s, renoise_steps=s - 1, cfg=(8.0, 8.0), **kw)
                for i, s in enumerate(steps_list)]
        ends = {}
        while eng.busy:
            done = eng.step()
            if done:
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                for q in done:
                    ends[id(q)] = e
        torch.cuda.synchronize()
        lat = [start.elapsed_time(ends[id(q)]) for q in reqs]
        return max(lat) / 1e3, lat

    def static_run(steps_list):
        """Requests grouped by step count into sample() calls of up to 64, all queued at t=0."""
        start = torch.cuda.Event(enable_timing=True)
        start.record()
        lat_ev = []
        by_steps = {}
        for i, s in enumerate(steps_list):
            by_steps.setdefault(s, []).append(i)
        for s in sorted(by_steps):
            idx = by_steps[s]
            for j in range(0, len(idx), MB):
                part = idx[j:j + MB]
                b = len(part)
                c = {k: v[[i % MB for i in part]] for k, v in cond.items()}
                u = {k: v[:b] for k, v in uncond.items()}
                U.sample(model, c, (b, H, H), u, steps=s, renoise_steps=s - 1, cfg=8.0, generator=gens(b, part[0]), **kw)
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                lat_ev += [e] * b
        torch.cuda.synchronize()
        lat = [start.elapsed_time(e) for e in lat_ev]
        return max(lat) / 1e3, lat

    arms = {"uniform_engine": lambda: engine_run([8] * N_UNI), "uniform_sample": lambda: static_run([8] * N_UNI),
            "mixed_engine": lambda: engine_run(mixed_steps), "mixed_static": lambda: static_run(mixed_steps)}
    n_img = {"uniform_engine": N_UNI, "uniform_sample": N_UNI, "mixed_engine": args.mixed, "mixed_static": args.mixed}
    for f in arms.values():           # warm-up: every shape the timed windows use
        f()
    rates = {k: [] for k in arms}
    p50 = {k: [] for k in arms}
    p95 = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, f in arms.items():
            sec, lat = f()
            lat.sort()
            rates[k].append(n_img[k] / sec)
            p50[k].append(lat[len(lat) // 2])
            p95[k].append(lat[min(len(lat) - 1, int(0.95 * len(lat)))])
    med = {k: statistics.median(v) for k, v in rates.items()}
    res = {"gpu": gpu_info(), "rounds": args.rounds, "latent": H, "max_batch": MB, "uniform_requests": N_UNI,
           "mixed_requests": args.mixed, "mixed_steps_hist": {s: mixed_steps.count(s) for s in (8, 12, 16)},
           "images_per_s": rates, "median_images_per_s": med,
           "spread_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
           "latency_ms_p50": p50, "latency_ms_p95": p95,
           "uniform_engine_vs_sample": med["uniform_engine"] / med["uniform_sample"],
           "mixed_engine_vs_static": med["mixed_engine"] / med["mixed_static"]}
    for k in arms:
        print(f"[bench_engine] {k}: {med[k]:.2f} img/s (rounds {', '.join(f'{r:.2f}' for r in rates[k])}), "
              f"p50 {statistics.median(p50[k]):.0f} ms, p95 {statistics.median(p95[k]):.0f} ms", file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
