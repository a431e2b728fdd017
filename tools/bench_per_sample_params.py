"""Cost of per-sample sampling settings, timed in one process with the modes alternating so that all see the same clocks and
neighbours:

  * `scalar` vs `per_sample`: the `sample` workload of bench.py (bs 64, 32x32, 8 steps, CFG) with scalar arguments and with
    all-equal per-sample tensors (cfg [B], temperature [B, 2], t_start / t_end [B]) -- the same tokens;
  * `sweep_batched` vs `sweep_split`: a 4-value cfg sweep of 16 images each, as one bs-64 call with per-sample cfg or as four
    bs-16 calls, one per value.

  python tools/bench_per_sample_params.py [--rounds 3] [--calls 3]

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
    ap.add_argument("--calls", type=int, default=3, help="sample() calls (or sweeps) per timed window")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    model = bench.build_model(dev)
    model.pack_weights()
    w = bench.WORKLOADS["sample"]
    B, H, steps = w["batch"], w["latent"], w["steps"]
    cond, uncond = synthetic_conditioning(B, bench.BYT5_LEN, with_clip_image=w["clip_image"], seed=1234, device=dev)
    kw = dict(steps=steps, renoise_steps=steps - 1)
    scalar = dict(temperature=(1.0, 0.2), cfg=8.0, t_start=1.0, t_end=0.0)
    per = dict(temperature=torch.tensor([[1.0, 0.2]] * B), cfg=torch.full((B,), 8.0), t_start=torch.ones(B), t_end=torch.zeros(B))
    sweep = [2.0, 4.0, 6.0, 8.0]
    n_per = B // len(sweep)
    sweep_cfg = torch.tensor(sweep).repeat_interleave(n_per)
    parts = [({k: v[j * n_per:(j + 1) * n_per] for k, v in cond.items()}, {k: v[j * n_per:(j + 1) * n_per] for k, v in uncond.items()})
             for j in range(len(sweep))]

    def run(mode):
        if mode == "scalar":
            return U.sample(model, cond, (B, H, H), uncond, **kw, **scalar)
        if mode == "per_sample":
            return U.sample(model, cond, (B, H, H), uncond, **kw, **per)
        if mode == "sweep_batched":
            return U.sample(model, cond, (B, H, H), uncond, cfg=sweep_cfg, temperature=(1.0, 0.2), **kw)
        return [U.sample(model, c, (n_per, H, H), u, cfg=v, temperature=(1.0, 0.2), **kw) for (c, u), v in zip(parts, sweep)]

    torch.manual_seed(0)
    a = run("scalar")
    torch.manual_seed(0)
    same_tokens = bool(torch.equal(a, run("per_sample")))
    modes = ("scalar", "per_sample", "sweep_batched", "sweep_split")
    for mode in modes:           # warm-up: every shape and kernel instantiation
        run(mode)
    torch.cuda.synchronize()
    rates = {m: [] for m in modes}
    for _ in range(args.rounds):
        for mode in modes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.calls):
                run(mode)
            e1.record()
            torch.cuda.synchronize()
            rates[mode].append(B * args.calls / (e0.elapsed_time(e1) / 1e3))
    med = {k: statistics.median(v) for k, v in rates.items()}
    res = {"gpu": gpu_info(), "rounds": args.rounds, "calls_per_window": args.calls, "batch": B, "latent": H, "steps": steps,
           "sweep_cfg": sweep, "images_per_s": rates, "median": med, "scalar_vs_per_sample_tokens_equal": same_tokens,
           "per_sample_cost_pct": 100.0 * (1.0 - med["per_sample"] / med["scalar"]),
           "sweep_batched_speedup": med["sweep_batched"] / med["sweep_split"]}
    for k in modes:
        print(f"[bench_per_sample_params] {k}: {med[k]:.2f} img/s (rounds {', '.join(f'{r:.2f}' for r in rates[k])})",
              file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
