"""Token scoring, timed in one process with the arms alternating, on the default model with L_byt5=128+clip:

  * fused: Paella.token_scores (features, then one fused out_mapper + log-softmax kernel), unguided and with cfg 4;
  * unfused: F.cross_entropy(model(...), targets, reduction='none') on the same inputs (the fp32 logits [B, 8192, H, W] reach
    HBM and ATen's log_softmax reads them back); with cfg the two forwards' logits are mixed first, as the notebook does;
  * score: utils.score with the default 8 levels, unguided, at bs 64 / 32x32.

The token_scores arms run at bs 64 / 32x32 and bs 16 / 64x64.  Each arm's peak is torch.cuda.max_memory_allocated over one call.
A separate torch.profiler run sums the device time of token_score_kernel and of the out_mapper GEMM (pb200_paella_logits) on the
same rows, one call each.

  python tools/bench_scores.py [--rounds 3]

Prints one JSON line with every round, medians and ranges, the peaks, the profiled kernel times, and the GPU name, power limit
and maximum SM clock of the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

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
    CFG = 4.0
    shapes = {"bs64_32x32": (64, 32), "bs16_64x64": (16, 64)}

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    def peak(f):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        f()
        torch.cuda.synchronize()
        return (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20

    res = {"gpu": gpu_info(), "rounds": args.rounds, "cfg": CFG, "shapes": {}}
    for name, (B, H) in shapes.items():
        cond, uncond = synthetic_conditioning(B, bench.BYT5_LEN, seed=1234, device=dev)
        g = torch.Generator().manual_seed(7)
        x = torch.randint(0, model.num_labels, (B, H, H), generator=g).to(dev)
        y = torch.randint(0, model.num_labels, (B, H, H), generator=g).to(dev)
        r = torch.rand(B, generator=g).to(dev)

        def fused(cfg):
            return lambda: model.token_scores(x, r, y, cond["byt5"], cond["clip"], cfg=cfg, unconditional_inputs=uncond if cfg else None)

        def unfused(cfg):
            def f():
                lc = model(x, r, cond["byt5"], cond["clip"])
                if cfg:
                    lc = lc * cfg + model(x, r, uncond["byt5"], uncond["clip"]) * (1 - cfg)
                return F.cross_entropy(lc, y, reduction="none")
            return f
        arms = {"fused": fused(None), "unfused": unfused(None), "fused_cfg": fused(CFG), "unfused_cfg": unfused(CFG)}
        if B == 64:
            gens = [torch.Generator(device=dev).manual_seed(i) for i in range(B)]
            arms["score_8_levels"] = lambda: U.score(model, y, cond, generator=gens)
        with torch.inference_mode():
            for f in arms.values():            # warm-up: every shape the timed windows use
                f()
            peaks = {a: peak(f) for a, f in arms.items()}
            rates = {a: [] for a in arms}
            for _ in range(args.rounds):
                for a, f in arms.items():
                    rates[a].append(B / timed(f))
            # device time of the scoring kernel against the out_mapper GEMM on the same rows, one profiled call each
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                arms["fused"]()
                arms["unfused"]()
                torch.cuda.synchronize()
        kern = {"token_score_kernel": 0.0, "out_mapper_gemm": 0.0}
        gemm_shape = None
        for e in prof.key_averages():
            if "token_score_kernel" in e.key:
                kern["token_score_kernel"] += e.device_time_total / 1e3
        # the out_mapper GEMM is the forward's last gemm_f16_kernel launch; take it from the raw events
        last_gemm = [ev for ev in prof.events() if "gemm_f16_kernel" in ev.name]
        if last_gemm:
            kern["out_mapper_gemm"] = last_gemm[-1].device_time_total / 1e3
            gemm_shape = last_gemm[-1].name[:80]
        med = {k: statistics.median(v) for k, v in rates.items()}
        res["shapes"][name] = {"batch": B, "latent": H, "images_per_s": rates, "median_images_per_s": med,
                               "range_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
                               "peak_mib": peaks, "profiled_device_ms": kern, "gemm_kernel": gemm_shape}
        for k in arms:
            print(f"[bench_scores] {name} {k}: {med[k]:.2f} img/s ({min(rates[k]):.2f}-{max(rates[k]):.2f}), peak {peaks[k]:.0f} MiB",
                  file=sys.stderr, flush=True)
        print(f"[bench_scores] {name} profiled ms {json.dumps(kern)}", file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
