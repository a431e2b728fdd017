"""Cost of per-sample attn_weights, timed in one process with the arms alternating so that all see the same clocks and
neighbours (default model, 32x32 latents, L_byt5=128+clip, CFG 8, temperature (1.0, 0.2), 8 steps):

  * `none` / `shared` / `per_sample`: the `sample` workload of bench.py (bs 64) through sample_notebook with no weights, one
    shared notebook vector (a device tensor), and the same vector for every sample as a per-sample list -- the last two must
    give the same tokens.  Also the `attention` kernel family's CUDA-event time of one profiled call per arm;
  * `mixed_batched` / `mixed_grouped`: 64 notebook-style requests with 4 prompt lengths (32, 64, 96, 128; 16 each), each with
    the notebook's vector for its length, as one call with per-sample vectors (prompts padded to the longest, as a batched
    tokenizer pads them) or as four calls grouped by length;
  * `engine_plain` / `engine_weighted`: tools/bench_engine.py's uniform load (256 requests of 8 steps, max_batch 64) without
    and with a per-request vector.

  python tools/bench_attn_weights.py [--rounds 3]

Prints one JSON line: images/s per arm and round, the medians, and the GPU name and power limit read in the same run.
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


def notebook_vec(n):
    """paella_inference.ipynb cell 7: 1.2 everywhere, 0.4 on the last 4 entries."""
    v = torch.full((n,), 1.2)
    v[-4:] = 0.4
    return v


def main():
    import bench
    from bench_per_sample_params import gpu_info
    from paella_b200 import _lib
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
    w = bench.WORKLOADS["sample"]
    B, H, steps, L = w["batch"], w["latent"], w["steps"], bench.BYT5_LEN
    cond, uncond = synthetic_conditioning(B, L, seed=1234, device=dev)
    kw = dict(steps=steps, renoise_steps=steps - 1, temperature=(1.0, 0.2), cfg=(8.0, 8.0))
    vec = notebook_vec(L)
    vec_d = vec.to(dev)
    lens = [32, 64, 96, 128]
    per_len = B // len(lens)
    mixed_vecs = [notebook_vec(n) for n in lens for _ in range(per_len)]
    groups = [({k: (v[j * per_len:(j + 1) * per_len, :n] if k == "byt5" else v[j * per_len:(j + 1) * per_len]) for k, v in cond.items()},
               {k: (v[j * per_len:(j + 1) * per_len, :n] if k == "byt5" else v[j * per_len:(j + 1) * per_len]) for k, v in uncond.items()},
               notebook_vec(n)) for j, n in enumerate(lens)]
    row = lambda d, i: {k: v[i:i + 1] for k, v in d.items()}          # noqa: E731
    N_UNI = 256
    eng = SamplingEngine(model, latent_hw=(H, H), max_batch=B, max_cond_len=L + 4, unconditional_inputs=row(uncond, 0))

    def engine_run(weighted):
        g = [torch.Generator(device=dev).manual_seed(i) for i in range(N_UNI)]
        for i in range(N_UNI):
            eng.submit(row(cond, i % B), generator=g[i], attn_weights=vec if weighted else None, **kw)
        eng.run_until_idle()

    arms = {
        "none": lambda: U.sample_notebook(model, cond, (B, H, H), uncond, **kw),
        "shared": lambda: U.sample_notebook(model, cond, (B, H, H), uncond, attn_weights=vec_d, **kw),
        "per_sample": lambda: U.sample_notebook(model, cond, (B, H, H), uncond, attn_weights=[vec] * B, **kw),
        "mixed_batched": lambda: U.sample_notebook(model, cond, (B, H, H), uncond, attn_weights=mixed_vecs, **kw),
        "mixed_grouped": lambda: [U.sample_notebook(model, c, (per_len, H, H), u, attn_weights=v.to(dev), **kw) for c, u, v in groups],
        "engine_plain": lambda: engine_run(False),
        "engine_weighted": lambda: engine_run(True),
    }
    n_img = {k: (N_UNI if k.startswith("engine") else B) for k in arms}

    torch.manual_seed(0)
    a = arms["shared"]()[0]
    torch.manual_seed(0)
    same_tokens = bool(torch.equal(a, arms["per_sample"]()[0]))
    for f in arms.values():           # warm-up: every shape the timed windows use
        f()
    torch.cuda.synchronize()
    rates = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, f in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            rates[k].append(n_img[k] / (e0.elapsed_time(e1) / 1e3))

    # one profiled call per sample_notebook arm (separate from the timed windows): the attention family's event time
    L_ = _lib.lib()
    attention_ms = {}
    for k in ("none", "shared", "per_sample", "mixed_batched"):
        L_.pb200_profile_enable(1)
        arms[k]()
        torch.cuda.synchronize()
        buf = ctypes.create_string_buffer(65536)
        _lib.check(L_.pb200_profile_report(buf, 65536), "profile_report")
        L_.pb200_profile_enable(0)
        prof = json.loads(buf.value.decode())
        attention_ms[k] = {"ms": round(prof["attention"]["ms"], 3), "launches": prof["attention"]["launches"]}

    med = {k: statistics.median(v) for k, v in rates.items()}
    res = {"gpu": gpu_info(), "rounds": args.rounds, "batch": B, "latent": H, "steps": steps, "byt5_len": L,
           "mixed_prompt_lengths": lens, "engine_requests": N_UNI, "images_per_s": rates, "median_images_per_s": med,
           "spread_images_per_s": {k: [min(v), max(v)] for k, v in rates.items()},
           "attention_family_ms_per_call": attention_ms, "shared_vs_per_sample_tokens_equal": same_tokens,
           "per_sample_vs_shared": med["per_sample"] / med["shared"],
           "mixed_batched_vs_grouped": med["mixed_batched"] / med["mixed_grouped"],
           "engine_weighted_vs_plain": med["engine_weighted"] / med["engine_plain"]}
    for k in arms:
        print(f"[bench_attn_weights] {k}: {med[k]:.2f} img/s (rounds {', '.join(f'{r:.2f}' for r in rates[k])})",
              file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
