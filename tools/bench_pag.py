"""Perturbed-attention guidance, timed in one process with the arms alternating:

  * ``sample()`` on the default model at bs 64, 32x32 latents, L_byt5=128+clip, CFG 8, 8 steps, per-sample generators (bench.py's
    ``sample`` shape), plain and with pag=2.0 (the default blocks) on every sample;
  * the same at bs 16, 64x64 latents, 12 steps (bench.py's ``sample64`` shape, without its CLIP-image conditioning);
  * one attention launch (pb200_attention_perturb) at the deepest level of a 32x32 guided batch (128 rows, 16 positions) and the
    level above it (64 positions), every row perturbed against pag_batch 0, with CUDA events over many launches.

A perturbed sample runs one more denoiser row per guided step, as one guidance prompt does, so the PAG arm is expected to cost
about 1.5x the plain arm's time.

  python tools/bench_pag.py [--rounds 3]

Prints one JSON line with every round, medians and ranges, and the GPU name, power limit and maximum SM clock of the same run.
"""
import argparse
import ctypes
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
    from paella_b200._lib import lib
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
        for arm, pag in (("plain", None), ("pag", [2.0] * B)):
            arms[f"{name}/{arm}"] = (B, lambda cond=cond, uncond=uncond, B=B, H=H, kw=kw, pag=pag:
                                     U.sample(model, cond, (B, H, H), uncond, generator=gens(B, 0), pag=pag, **kw))
    rates = {a: [] for a in arms}
    for a, (_, f) in arms.items():          # warm-up: every shape the timed windows use
        f()
    for _ in range(args.rounds):
        for a, (B, f) in arms.items():
            rates[a].append(B / timed(f))

    # one attention launch, every row perturbed vs none
    L = lib()
    att = {}
    for P in (16, 64):
        Bt, E, nh, S = 128, 1280, 16, bench.BYT5_LEN + 77
        qkv = (torch.randn(Bt * P, 3 * E, device=dev) * 0.5).half()
        ckv = (torch.randn(Bt, S, 2 * E, device=dev) * 0.5).half()
        out = torch.empty(Bt * P, E, dtype=torch.float16, device=dev)
        masks = torch.full((Bt,), 1, dtype=torch.int64, device=dev)
        vp = lambda x: ctypes.c_void_p(x.data_ptr())        # noqa: E731

        def launch(n_pag):
            return L.pb200_attention_perturb(vp(qkv), vp(ckv), None, None, Bt, vp(out), Bt, P, S, E, nh, 1, None, 0, 0, None, None,
                                             0, None, None, None, 0, 0, None, None, None, 0, None, 0, vp(masks), n_pag, 0, None)
        res = {}
        for arm, n_pag in (("plain", 0), ("pag", Bt)):
            for _ in range(10):
                assert launch(n_pag) == 0
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(200):
                launch(n_pag)
            e1.record()
            torch.cuda.synchronize()
            res[arm] = e0.elapsed_time(e1) / 200 * 1e3
        att[f"P{P}"] = {"us_per_launch": res, "pag_over_plain": res["pag"] / res["plain"]}

    med = {k: statistics.median(v) for k, v in rates.items()}
    out = {"gpu": gpu_info(), "rounds": args.rounds, "images_per_s": rates, "median_images_per_s": med,
           "range_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
           "time_pag_over_plain": {n: med[f"{n}/plain"] / med[f"{n}/pag"] for n in shapes}, "attention": att}
    for k in rates:
        print(f"[bench_pag] {k}: {med[k]:.2f} img/s ({min(rates[k]):.2f}-{max(rates[k]):.2f})", file=sys.stderr, flush=True)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
