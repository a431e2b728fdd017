"""Cost of the batch-invariant mode (Paella.batch_invariant) and of the engine's batched conditioning admission, every arm
alternated ``--rounds`` times in one process so that all see the same clocks and neighbours:

  * the `sample` (bs 64, 32x32, 8 steps, CFG) and `sample64` (bs 16, 64x64, 12 steps, CFG) workloads of bench.py, mode off
    vs on: images/s, and whether the two modes give the same tokens from the same seed;
  * GPU time to write the conditioning of 64 admitted requests (L_byt5 = 128 + clip, own unconditional rows) into an engine
    cache: one write_conditioning per request and slot vs one per run of contiguous slots with one layout (engine.admission_runs);
  * tools/bench_engine.py's uniform load (256 requests of 8 steps at t=0, max_batch 64) with per-request and with batched
    admission.

  python tools/bench_batch_invariant.py [--rounds 3] [--calls 2]

Prints one JSON line: per arm the rounds, median and range, and the GPU name and power limit read in the same run.
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


def _summary(v):
    return {"rounds": v, "median": statistics.median(v), "range": [min(v), max(v)]}


def _timed(f):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3, out


def main():
    import bench
    from bench_generators import gpu_info
    from paella_b200 import engine as E
    from paella_b200 import utils as U
    from paella_b200.synth import synthetic_conditioning
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=2, help="sample() calls per timed window")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    model = bench.build_model(dev)
    model.pack_weights()
    res = {"gpu": gpu_info(), "rounds": args.rounds, "workloads": {}}

    # ---- sample / sample64, mode off vs on
    for name in ("sample", "sample64"):
        w = bench.WORKLOADS[name]
        B, H, steps = w["batch"], w["latent"], w["steps"]
        cond, uncond = synthetic_conditioning(B, bench.BYT5_LEN, with_clip_image=w["clip_image"], seed=1234, device=dev)
        kw = dict(steps=steps, renoise_steps=steps - 1, temperature=(1.0, 0.2), cfg=8.0)

        def run(on):
            model.batch_invariant = on
            torch.manual_seed(1234)
            return U.sample(model, cond, (B, H, H), uncond, **kw)

        toks = {on: run(on) for on in (False, True)}          # warm-up, and the tokens of each mode
        rates = {False: [], True: []}
        for _ in range(args.rounds):
            for on in (False, True):
                sec, _ = _timed(lambda: [run(on) for _ in range(args.calls)])
                rates[on].append(B * args.calls / sec)
        off, on = statistics.median(rates[False]), statistics.median(rates[True])
        res["workloads"][name] = {"batch": B, "latent": H, "steps": steps, "images_per_s_off": _summary(rates[False]),
                                  "images_per_s_on": _summary(rates[True]), "mode_on_cost_pct": 100.0 * (1.0 - on / off),
                                  "tokens_equal": bool(torch.equal(toks[False], toks[True])),
                                  "tokens_differing": int((toks[False] != toks[True]).sum()), "tokens": toks[False].numel()}
        print(f"[bench_batch_invariant] {name}: off {off:.2f} img/s, on {on:.2f} img/s", file=sys.stderr, flush=True)
    model.batch_invariant = False

    # ---- admission of 64 requests: per-request vs batched conditioning projection
    H, MB = 32, 64
    cond, uncond = synthetic_conditioning(MB, bench.BYT5_LEN, seed=1234, device=dev)
    row = lambda d, i: {k: v[i:i + 1] for k, v in d.items()}          # noqa: E731
    eng = E.SamplingEngine(model, latent_hw=(H, H), max_batch=MB, max_cond_len=bench.BYT5_LEN + 4)
    writes = [(i, row(cond, i)) for i in range(MB)] + [(MB + i, row(uncond, i)) for i in range(MB)]

    def admit_per_request():
        for slot, x in writes:
            model.write_conditioning(eng.cache, slot, x, (H, H))

    def admit_batched():
        for run in E.admission_runs([(slot, E.cond_layout(x)) for slot, x in writes]):
            model.write_conditioning(eng.cache, writes[run[0]][0], E._cat_inputs([writes[i][1] for i in run], dev), (H, H))

    arms = {"per_request": admit_per_request, "batched": admit_batched}
    with torch.inference_mode():
        for f in arms.values():
            f()
        torch.cuda.synchronize()
        ms = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, f in arms.items():
                ms[k].append(_timed(f)[0] * 1e3)
    res["admit_64_requests_ms"] = {k: _summary(v) for k, v in ms.items()}
    print(f"[bench_batch_invariant] admit 64: per-request {statistics.median(ms['per_request']):.1f} ms, "
          f"batched {statistics.median(ms['batched']):.1f} ms", file=sys.stderr, flush=True)

    # ---- engine uniform load with per-request and batched admission
    N_UNI = 256
    eng = E.SamplingEngine(model, latent_hw=(H, H), max_batch=MB, max_cond_len=bench.BYT5_LEN + 4, unconditional_inputs=row(uncond, 0))
    batched_runs = E.admission_runs

    def engine_run(batched):
        E.admission_runs = batched_runs if batched else (lambda w: [[i] for i in sorted(range(len(w)), key=lambda i: w[i][0])])
        try:
            g = [torch.Generator(device=dev).manual_seed(i) for i in range(N_UNI)]

            def go():
                for i in range(N_UNI):
                    eng.submit(row(cond, i % MB), generator=g[i], steps=8, renoise_steps=7, cfg=(8.0, 8.0), temperature=(1.0, 0.2))
                eng.run_until_idle()
            return N_UNI / _timed(go)[0]
        finally:
            E.admission_runs = batched_runs

    for b in (False, True):
        engine_run(b)
    rates = {"per_request": [], "batched": []}
    for _ in range(args.rounds):
        for b, k in ((False, "per_request"), (True, "batched")):
            rates[k].append(engine_run(b))
    res["engine_uniform_images_per_s"] = {k: _summary(v) for k, v in rates.items()}
    print(f"[bench_batch_invariant] engine uniform: per-request admission {statistics.median(rates['per_request']):.2f} img/s, "
          f"batched {statistics.median(rates['batched']):.2f} img/s", file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
