"""Guidance prompts, timed in one process with the arms alternating: ``sample()`` on the default model at bs 64, 32x32 latents,
L_byt5=128+clip, CFG 8, temperature (1.0, 0.2), 8 steps, per-sample generators (the shape of bench.py's ``sample`` workload):

  * no terms;
  * 1 term per sample (weight 0.5);
  * 2 terms per sample (weights 0.5 and -0.5, the second a further negative prompt).

Every term prompt has the base prompt's layout.  A guided step runs 2 + J denoiser rows per sample instead of 2, sharing the
conditioning-free prefix, so a J-term arm is expected to cost about (2 + J) / 2 of the plain arm's forward time.  Then the
guidance_mix kernel alone is timed with CUDA events over many launches on the 2-term arm's shapes, and its bytes (read 2 + J
fp32 rows, write one, per composed sample) are set against the H100 SXM's 3.35 TB/s data-sheet HBM bandwidth.

  python tools/bench_guidance_prompts.py [--rounds 3]

Prints one JSON line with every round, medians and ranges, the mix kernel's time and bandwidth, and the GPU name, power limit
and maximum SM clock of the same run.
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

HBM_BYTES_PER_S = 3.35e12        # H100 SXM data sheet


def main():
    import bench
    from bench_per_sample_params import gpu_info
    from paella_b200 import ops
    from paella_b200 import utils as U
    from paella_b200._lib import check, current_stream, lib, ptr
    from paella_b200.synth import synthetic_conditioning
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    model = bench.build_model(dev)
    model.pack_weights()
    H, B, STEPS = 32, 64, 8
    cond, uncond = synthetic_conditioning(B, bench.BYT5_LEN, seed=1234, device=dev)
    extra, _ = synthetic_conditioning(2 * B, bench.BYT5_LEN, seed=4321, device=dev)
    row = lambda d, i: {k: v[i:i + 1] for k, v in d.items()}          # noqa: E731
    kw = dict(temperature=(1.0, 0.2), steps=STEPS, renoise_steps=STEPS - 1, cfg=8.0)
    weights = {"no terms": [], "1 term": [0.5], "2 terms": [0.5, -0.5]}
    terms = {a: [[(row(extra, 2 * b + j), w) for j, w in enumerate(ws)] for b in range(B)] if ws else None
             for a, ws in weights.items()}

    def gens(n, base):
        return [torch.Generator(device=dev).manual_seed(base + i) for i in range(n)]

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    def run(a):
        return lambda: U.sample(model, cond, (B, H, H), uncond, generator=gens(B, 0), guidance_prompts=terms[a], **kw)

    rates = {a: [] for a in weights}
    for a in weights:                          # warm-up: every shape the timed windows use
        run(a)()
    for _ in range(args.rounds):
        for a in weights:
            rates[a].append(B / timed(run(a)))

    # the mix kernel alone, on the 2-term arm's shapes: 4B rows of features, B composed samples
    J, c_out, hw = 2, model._cfg["c_out"], H * H
    feats = torch.randn((4 * B) * hw, c_out, device=dev)
    rows, coef = ops.guidance_mix_table([weights["2 terms"]] * B, list(range(B)), [B + b for b in range(B)],
                                        [[2 * B + J * b + j for j in range(J)] for b in range(B)], [[8.0] * B])
    rows_d, coef_d = ops.to_device_packed([rows, coef[0]], dev)
    model.guidance_mix(feats, hw, rows_d, coef_d)

    def launch():        # the C entry point itself: Paella.guidance_mix's weight-version check costs more host time than the kernel
        check(lib().pb200_paella_guidance_mix(model._handle, ptr(feats), hw, ptr(rows_d), ptr(coef_d), B, 2 + J, current_stream()),
              "pb200_paella_guidance_mix")
    for _ in range(10):
        launch()
    n_launch = 200
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n_launch):
        launch()
    e1.record()
    torch.cuda.synchronize()
    mix_s = e0.elapsed_time(e1) / 1e3 / n_launch
    mix_bytes = B * hw * c_out * 4 * (2 + J + 1)

    med = {k: statistics.median(v) for k, v in rates.items()}
    res = {"gpu": gpu_info(), "rounds": args.rounds, "batch": B, "latent": H, "steps": STEPS,
           "images_per_s": rates, "median_images_per_s": med, "range_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
           "relative_to_no_terms": {k: med["no terms"] / v for k, v in med.items()},
           "guidance_mix": {"us_per_launch": mix_s * 1e6, "bytes": mix_bytes, "bytes_per_s": mix_bytes / mix_s,
                            "share_of_hbm_datasheet": mix_bytes / mix_s / HBM_BYTES_PER_S}}
    for k in rates:
        print(f"[bench_guidance_prompts] {k}: {med[k]:.2f} img/s ({min(rates[k]):.2f}-{max(rates[k]):.2f})", file=sys.stderr, flush=True)
    print(f"[bench_guidance_prompts] guidance_mix: {mix_s * 1e6:.1f} us, {mix_bytes / mix_s / 1e12:.2f} TB/s", file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
