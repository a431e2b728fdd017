"""Cost of per-sample generators: the `sample` (bs 64, 32x32, 8 steps, CFG) and `sample64` (bs 16, 64x64, 12 steps, CFG)
workloads of bench.py, timed with the default generator and with one generator per sample, alternating the two modes in
one process so that both see the same clocks and neighbours.

  python tools/bench_generators.py [--rounds 3] [--steps 3] [--workloads sample sample64]

Prints one JSON line: images/s per mode and round, the median of each, and the GPU name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_max_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # noqa: BLE001
        info["power_limit"] = f"unavailable ({type(e).__name__})"
    return info


def main():
    import bench
    from paella_b200 import utils as U
    from paella_b200.synth import synthetic_conditioning
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3, help="sample() calls per timed window")
    ap.add_argument("--workloads", nargs="+", default=["sample", "sample64"])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    model = bench.build_model(dev)
    model.pack_weights()
    res = {"gpu": gpu_info(), "rounds": args.rounds, "calls_per_window": args.steps, "workloads": {}}
    for name in args.workloads:
        w = bench.WORKLOADS[name]
        B, H, steps = w["batch"], w["latent"], w["steps"]
        cond, uncond = synthetic_conditioning(B, bench.BYT5_LEN, with_clip_image=w["clip_image"], seed=1234, device=dev)
        kw = dict(steps=steps, renoise_steps=steps - 1, temperature=(1.0, 0.2), cfg=8.0)
        gens = [torch.Generator(device=dev).manual_seed(1234 + i) for i in range(B)]

        def run(mode):
            if mode == "default":
                return U.sample(model, cond, (B, H, H), uncond, **kw)
            return U.sample(model, cond, (B, H, H), uncond, generator=gens, **kw)

        for mode in ("default", "per_sample"):       # warm-up: every shape and both kernel instantiations
            run(mode)
        torch.cuda.synchronize()
        rates = {"default": [], "per_sample": []}
        for _ in range(args.rounds):
            for mode in ("default", "per_sample"):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    run(mode)
                e1.record()
                torch.cuda.synchronize()
                rates[mode].append(B * args.steps / (e0.elapsed_time(e1) / 1e3))
        med = {k: statistics.median(v) for k, v in rates.items()}
        res["workloads"][name] = {"batch": B, "latent": H, "steps": steps, "images_per_s": rates, "median": med,
                                  "per_sample_cost_pct": 100.0 * (1.0 - med["per_sample"] / med["default"])}
        print(f"[bench_generators] {name}: default {med['default']:.2f} img/s, per-sample {med['per_sample']:.2f} img/s",
              file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
