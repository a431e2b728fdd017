"""LoRA adapters per sample, timed in one process with the arms alternating: 8-step CFG sample() at bs 64 / 32x32 on the default
model with L_byt5=128+clip (bench.py's `sample` workload), arms

  * none:       no adapter (the bench.py path);
  * one_r16:    every sample on one rank-16 adapter covering every AttnBlock's in_proj, out_proj and kv_mapper;
  * eight_r16:  eight distinct rank-16 adapters, sample i on adapter i % 8;
  * one_r64:    every sample on one rank-64 adapter;
  * merged:     the rank-16 adapter folded into a second model's weights with merge_lora (the single-model alternative);
  * half_r16:   half the samples on the rank-16 adapter, the others on none;
  * engine_none, engine_half_r16: a SamplingEngine (max_batch 64) given the same 64 prompts as 64 requests, 8 steps each, without
                adapters and with every other request on the rank-16 adapter, drained with run_until_idle (the engine's default
                temperature (0.7, 0.3) and cfg (8, 8); its unconditional slot is engine-wide, a request with an adapter gets its own).

Each arm is warmed up, then timed `--rounds` times with device synchronisation (CUDA events), rounds alternating between arms.
A separate torch.profiler run of one one_r16 call sums the device time of the shrink and expand launches; their algorithmic bytes (each
adapted row's input read once and its output read and written once: 14c bytes per in_proj row, 10c per out_proj row) over that
time gives the achieved bandwidth, against the 3.35 TB/s of the H100 SXM data sheet.

  python tools/bench_lora.py [--rounds 3]

Prints one JSON line with every round, medians and ranges, the profiled kernel time and bytes, and the GPU name, power limit and
maximum SM clock of the same run.
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

HBM_BYTES_PER_S = 3.35e12


def adapter_sd(cfg, rank, seed):
    from paella_b200.lora import served_targets
    g = torch.Generator().manual_seed(seed)
    out = {}
    for mod, (_, _, fin, fout) in served_targets(cfg).items():
        out[mod + ".lora_A.weight"] = torch.randn(rank, fin, generator=g) / fin ** 0.5
        out[mod + ".lora_B.weight"] = torch.randn(fout, rank, generator=g) * 0.02
    return out


def lora_bytes_per_call(model, B, H, steps):
    """Algorithmic bytes of the shrink and expand launches in the AttnBlocks of one guided sample() call (every row adapted)."""
    c = model._cfg
    total = 0
    for lvl, (kinds, n) in enumerate(zip(c["level_config"], c["blocks"])):
        if "A" not in kinds:
            continue
        P = ((H // c["patch_size"]) >> lvl) ** 2
        ch = c["c_hidden"][lvl]
        rows = 2 * B * P * kinds.count("A") * n * 2          # CFG pair rows, down and up path
        total += rows * (14 * ch + 10 * ch)
    return total * steps


def main():
    import bench
    from bench_per_sample_params import gpu_info
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    from paella_b200.lora import load_lora, merge_lora
    from paella_b200.synth import synthetic_conditioning
    from torch.profiler import ProfilerActivity, profile
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    model = bench.build_model(dev)
    model.pack_weights()
    B, H, steps = 64, 32, 8
    cond, uncond = synthetic_conditioning(B, bench.BYT5_LEN, seed=1234, device=dev)
    sd16 = adapter_sd(model._cfg, 16, 1)
    a16 = load_lora(model, sd16)
    a64 = load_lora(model, adapter_sd(model._cfg, 64, 2))
    eight = [a16] + [load_lora(model, adapter_sd(model._cfg, 16, 10 + i)) for i in range(7)]
    merged = bench.build_model(dev)
    merged.load_state_dict(merge_lora(model.state_dict(), sd16))
    merged.pack_weights()

    def run(m, lora):
        return lambda: U.sample(m, cond, (B, H, H), uncond, steps=steps, renoise_steps=steps - 1, lora=lora)
    eng = SamplingEngine(model, latent_hw=(H, H), max_batch=B, max_cond_len=bench.BYT5_LEN + 4,
                         unconditional_inputs={k: v[:1] for k, v in uncond.items()})

    def run_engine(lora):
        def f():
            for i in range(B):
                eng.submit({k: v[i:i + 1] for k, v in cond.items()}, generator=torch.Generator(device=dev).manual_seed(i),
                           steps=steps, lora=lora[i])
            eng.run_until_idle()
        return f
    arms = {"none": run(model, None), "one_r16": run(model, a16), "eight_r16": run(model, [eight[i % 8] for i in range(B)]),
            "one_r64": run(model, a64), "merged": run(merged, None), "half_r16": run(model, [a16 if i % 2 else None for i in range(B)]),
            "engine_none": run_engine([None] * B), "engine_half_r16": run_engine([a16 if i % 2 else None for i in range(B)])}

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    res = {"gpu": gpu_info(), "rounds": args.rounds, "batch": B, "latent": H, "steps": steps}
    with torch.inference_mode():
        for f in arms.values():
            f()
            f()
        torch.cuda.synchronize()
        rates = {a: [] for a in arms}
        for _ in range(args.rounds):
            for a, f in arms.items():
                rates[a].append(B / timed(f))
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            arms["one_r16"]()
            torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        for name in ("lora_shrink_kernel", "lora_expand_kernel"):
            if name in e.key:
                ms, n = kern.get(name, (0.0, 0))
                kern[name] = (ms + e.device_time_total / 1e3, n + e.count)
    lora_ms = sum(ms for ms, _ in kern.values())
    n_launch = sum(n for _, n in kern.values())
    nbytes = lora_bytes_per_call(model, B, H, steps)
    med = {k: statistics.median(v) for k, v in rates.items()}
    res.update({"images_per_s": rates, "median_images_per_s": med, "range_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
                "cost_vs_none": {k: med["none"] / v - 1.0 for k, v in med.items()},
                "profiled_one_r16": {"lora_kernel_ms_per_call": lora_ms, "launches": n_launch, "by_kernel_ms_launches": kern,
                                     "algorithmic_bytes": nbytes,
                                     "achieved_bytes_per_s": nbytes / (lora_ms / 1e3) if lora_ms else None,
                                     "share_of_hbm_datasheet": nbytes / (lora_ms / 1e3) / HBM_BYTES_PER_S if lora_ms else None}})
    for k in arms:
        print(f"[bench_lora] {k}: {med[k]:.2f} img/s ({min(rates[k]):.2f}-{max(rates[k]):.2f})", file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
