"""Top-k / top-p truncation, timed in one process with the arms alternating, on two loads (default model, 32x32 latents,
L_byt5=128+clip, CFG 8, temperature (1.0, 0.2), 8 steps):

  * sample: ``sample()`` at bs 64 with per-sample generators (the shape of bench.py's ``sample`` workload);
  * engine: 256 requests through SamplingEngine, max_batch 64 (tools/bench_engine.py's uniform load).

Arms: ``none``; ``k_forced``: k = num_labels through the truncation kernels (every code kept: their pure overhead; the public
API turns k >= num_labels off, so this arm builds the table itself); ``top_k64``; ``top_p0.9``; ``half``: every other
sample with top_k=64, top_p=0.9.  One profiled call per arm gives the fused sampler family's event time.

  python tools/bench_truncation.py [--rounds 3]

Prints one JSON line with every round, medians and ranges, the GPU name, power limit and maximum SM clock, and the SM clock
read after every timed window, all from the same run.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    import bench
    from bench_per_sample_params import gpu_info
    from paella_b200 import _lib, ops
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
    NL = model.num_labels
    H, B, N, STEPS = 32, 64, 256, 8
    cond, uncond = synthetic_conditioning(B, bench.BYT5_LEN, seed=1234, device=dev)
    row = lambda d, i: {k: v[i:i + 1] for k, v in d.items()}          # noqa: E731
    kw = dict(temperature=(1.0, 0.2), steps=STEPS, renoise_steps=STEPS - 1)
    half_k = torch.tensor([64 if i % 2 else 0 for i in range(B)])
    half_p = torch.tensor([0.9 if i % 2 else 1.0 for i in range(B)], dtype=torch.float64)
    arms_kw = {"none": {}, "k_forced": {"top_k": NL}, "top_k64": {"top_k": 64}, "top_p0.9": {"top_p": 0.9},
               "half": {"top_k": half_k, "top_p": half_p}}
    real_table = ops.truncation_table

    def forced_table(top_k, top_p, batch, num_labels):      # k = num_labels kept in the table (the kernels' overhead)
        if isinstance(top_k, int) and top_k == num_labels and top_p is None:
            return torch.full((batch,), num_labels, dtype=torch.int32), torch.ones(batch)
        return real_table(top_k, top_p, batch, num_labels)

    def sm_clock():       # the SM clock right now (read-only query), next to the maximum in gpu_info
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
        return q or "unavailable"

    eng = SamplingEngine(model, latent_hw=(H, H), max_batch=B, max_cond_len=bench.BYT5_LEN + 4, unconditional_inputs=row(uncond, 0))

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
        return lambda: U.sample(model, cond, (B, H, H), uncond, cfg=8.0, generator=gens(B, 0), **kw, **arms_kw[a])

    def engine_run(a):
        def f():
            g = gens(N, 0)
            for i in range(N):
                tk = arms_kw[a].get("top_k")
                tp = arms_kw[a].get("top_p")
                if torch.is_tensor(tk):
                    tk, tp = int(tk[i % B]), float(tp[i % B])
                eng.submit(row(cond, i % B), generator=g[i], cfg=(8.0, 8.0), top_k=tk, top_p=tp, **kw)
            eng.run_until_idle()
        return f

    loads = {"sample": (sample_run, B), "engine": (engine_run, N)}
    rates = {f"{ld}/{a}": [] for ld in loads for a in arms_kw}
    clocks = {k: [] for k in rates}          # the SM clock read right after each timed window
    ops.truncation_table = forced_table
    try:
        for ld, (mk, _) in loads.items():          # warm-up: every shape the timed windows use
            for a in arms_kw:
                mk(a)()
        for _ in range(args.rounds):
            for ld, (mk, n) in loads.items():
                for a in arms_kw:
                    rates[f"{ld}/{a}"].append(n / timed(mk(a)))
                    clocks[f"{ld}/{a}"].append(sm_clock())
        # one profiled call per arm (separate from the timed windows): the fused sampler family's event time
        L_ = _lib.lib()
        sampler_ms = {}
        for ld, (mk, _) in loads.items():
            for a in arms_kw:
                L_.pb200_profile_enable(1)
                mk(a)()
                torch.cuda.synchronize()
                buf = ctypes.create_string_buffer(65536)
                _lib.check(L_.pb200_profile_report(buf, 65536), "profile_report")
                L_.pb200_profile_enable(0)
                prof = json.loads(buf.value.decode())
                fs = prof.get("fused_sampler", {"ms": 0.0, "launches": 0})
                sampler_ms[f"{ld}/{a}"] = {"ms": round(fs["ms"], 3), "launches": fs["launches"]}
    finally:
        ops.truncation_table = real_table
    med = {k: statistics.median(v) for k, v in rates.items()}
    res = {"gpu": gpu_info(), "rounds": args.rounds, "batch": B, "latent": H, "steps": STEPS, "engine_requests": N,
           "images_per_s": rates, "median_images_per_s": med, "range_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
           "fused_sampler_ms_per_call": sampler_ms, "sm_clock_after_each_window": clocks}
    for k in rates:
        print(f"[bench_truncation] {k}: {med[k]:.2f} img/s ({min(rates[k]):.2f}-{max(rates[k]):.2f}); fused sampler "
              f"{sampler_ms[k]['ms']:.1f} ms / {sampler_ms[k]['launches']} launches", file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
