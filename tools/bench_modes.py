"""Per-request sampling modes, timed in one process with the arms alternating (default model, 32x32 latents, L_byt5=128+clip,
CFG 8, temperature (1.0, 0.2), 8 steps, 256 requests, max_batch 64):

  * engine_multinomial: every request multinomial (the load of tools/bench_engine.py's uniform arm);
  * engine_mixed: the same requests, a quarter of them with sampling_quant_steps=6 (steps 6 and 7 in 'quant');
  * notebook_grouped: the mixed requests as sample_notebook calls of up to 64 grouped by mode, per-sample generators.

  python tools/bench_modes.py [--rounds 3]

Prints one JSON line with every round, the medians and the spread, and the GPU name and power limit read in the same run.
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
    from paella_b200.vqgan import VQModel
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    model = bench.build_model(dev)
    model.pack_weights()
    torch.manual_seed(0)
    vq = VQModel().to(dev).eval()
    H, MB, N, STEPS = 32, 64, 256, 8
    cond, uncond = synthetic_conditioning(MB, bench.BYT5_LEN, seed=1234, device=dev)
    row = lambda d, i: {k: v[i:i + 1] for k, v in d.items()}          # noqa: E731
    kw = dict(temperature=(1.0, 0.2), cfg=(8.0, 8.0), steps=STEPS, renoise_steps=STEPS - 1)
    quant = [i % 4 == 3 for i in range(N)]                             # a quarter switch to 'quant' at step 6
    eng = SamplingEngine(model, latent_hw=(H, H), max_batch=MB, max_cond_len=bench.BYT5_LEN + 4, unconditional_inputs=row(uncond, 0),
                         vqmodel=vq)

    def gens(n, base):
        return [torch.Generator(device=dev).manual_seed(base + i) for i in range(n)]

    def engine_run(mixed):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        g = gens(N, 0)
        for i in range(N):
            eng.submit(row(cond, i % MB), generator=g[i], sampling_quant_steps=6 if mixed and quant[i] else None, **kw)
        eng.run_until_idle()
        end.record()
        torch.cuda.synchronize()
        return start.elapsed_time(end) / 1e3

    def notebook_run():
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for q in (False, True):
            idx = [i for i in range(N) if quant[i] == q]
            for j in range(0, len(idx), MB):
                part = idx[j:j + MB]
                b = len(part)
                c = {k: v[[i % MB for i in part]] for k, v in cond.items()}
                u = {k: v[:b] for k, v in uncond.items()}
                U.sample_notebook(model, c, (b, H, H), u, sampling_quant_steps=6 if q else None, vqmodel=vq, generator=gens(b, part[0]),
                                  **kw)
        end.record()
        torch.cuda.synchronize()
        return start.elapsed_time(end) / 1e3

    arms = {"engine_multinomial": lambda: engine_run(False), "engine_mixed": lambda: engine_run(True), "notebook_grouped": notebook_run}
    for f in arms.values():           # warm-up: every shape the timed windows use
        f()
    rates = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, f in arms.items():
            rates[k].append(N / f())
    med = {k: statistics.median(v) for k, v in rates.items()}
    res = {"gpu": gpu_info(), "rounds": args.rounds, "latent": H, "max_batch": MB, "requests": N, "steps": STEPS,
           "images_per_s": rates, "median_images_per_s": med, "spread_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
           "engine_mixed_vs_notebook_grouped": med["engine_mixed"] / med["notebook_grouped"]}
    for k in arms:
        print(f"[bench_modes] {k}: {med[k]:.2f} img/s (rounds {', '.join(f'{r:.2f}' for r in rates[k])})", file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
