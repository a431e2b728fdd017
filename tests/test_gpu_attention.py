"""Attention core (ref/src/modules.py:12-19, ref/utils/alter_attention.py:19-36) through the C ABI (pb200_attention) against an
fp32 torch restatement on the same fp16-rounded q/k/v: the shapes of BASELINE configs 2 and 4, the shapes with ragged or
shared conditioning and ring wrap-around, and other head dims.  head_dim 80 runs the wgmma + TMA kernel (csrc/attention_wg.cu) by
default; PB200_ATTN_MMA_SYNC=1 (child process) sends it to the flash-style mma.sync kernel (csrc/attention.cu), which every
other head dim runs, so both kernels stay covered on every shape."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _log(payload):
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "attention_parity.jsonl"), "a") as f:
        f.write(json.dumps(payload) + "\n")


def _reference(qkv, ckv, kv_len, B, P, S, E, H, self_attn, aw):
    hd = E // H
    q = qkv[:, :E].float().view(B, P, H, hd).permute(0, 2, 1, 3)
    ks = qkv[:, E:2 * E].float().view(B, P, H, hd).permute(0, 2, 1, 3)
    vs = qkv[:, 2 * E:].float().view(B, P, H, hd).permute(0, 2, 1, 3)
    kc = ckv[:, :, :E].float().view(B, S, H, hd).permute(0, 2, 1, 3)
    vc = ckv[:, :, E:].float().view(B, S, H, hd).permute(0, 2, 1, 3)
    out = torch.empty(B, H, P, hd, device=qkv.device)
    for b in range(B):
        n = int(kv_len[b]) if kv_len is not None else S
        k = torch.cat([ks[b], kc[b, :, :n]], dim=1) if self_attn else kc[b, :, :n]
        v = torch.cat([vs[b], vc[b, :, :n]], dim=1) if self_attn else vc[b, :, :n]
        w = torch.softmax(q[b] @ k.transpose(1, 2) / hd ** 0.5, dim=-1)
        if aw is not None:
            w = w.clone()
            w[:, :, -aw.numel():] *= aw
        out[b] = w @ v
    return out.permute(0, 2, 1, 3).reshape(B * P, E)


def _run(B, P, S, H, hd, self_attn, varlen, weighted, seed=0):
    from paella_b200 import _lib
    L = _lib.lib()
    E = H * hd
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = (torch.randn(B * P, 3 * E, device=DEV, generator=g) * 1.5).half()
    ckv = (torch.randn(B, S, 2 * E, device=DEV, generator=g) * 1.5).half()
    kv_len = None
    if varlen:
        kv_len = torch.randint(max(1, S // 2), S + 1, (B,), device=DEV, generator=g, dtype=torch.int32)
        kv_len[0] = S
        for b in range(B):          # rows past a sample's length hold junk the kernel must ignore (finite, as the model guarantees)
            ckv[b, int(kv_len[b]):] = 777.0
    aw = (torch.rand(5, device=DEV, generator=g) * 2).float() if weighted else None
    out = torch.full((B * P, E), float("nan"), device=DEV, dtype=torch.float16)
    _lib.check(L.pb200_attention(_lib.ptr(qkv), _lib.ptr(ckv), _lib.ptr(kv_len), _lib.ptr(out), B, P, S, E, H, int(self_attn),
                                 _lib.ptr(aw), 5 if weighted else 0, B, _lib.current_stream()), "pb200_attention")
    torch.cuda.synchronize()
    want = _reference(qkv, ckv, kv_len, B, P, S, E, H, self_attn, aw)
    d = out.float() - want
    mx = float(d.abs().nan_to_num(1e9).max())
    if not (mx < 4e-3):          # layout diagnostics for a wrong kernel: error per (16-row block, 16-column block) of sample 0 / head 0,
        lines = [f"case B={B} P={P} S={S} H={H} hd={hd} self={self_attn} varlen={varlen} weighted={weighted}: max {mx:.3e}"]      # and per (sample, head)
        e = d.abs().nan_to_num(9.0).view(B, P, H, hd)
        lines.append("per (sample, head) max: " + " ".join(f"{float(e[b, :, h].max()):.1e}" for b in range(min(B, 4)) for h in range(min(H, 4))))
        blk = e[0, :, 0]
        for r0 in range(0, P, 16):
            lines.append(f"rows {r0:3d}+16: " + " ".join(f"{float(blk[r0:r0 + 16, c0:c0 + 16].max()):.1e}" for c0 in range(0, hd, 16)))
        lines.append("nan count: %d" % int(torch.isnan(out.float()).sum()))
        lines.append("got[0,:4,:6]  " + str(out.float().view(B, P, H, hd)[0, :4, 0, :6].tolist()))
        lines.append("want[0,:4,:6] " + str(want.view(B, P, H, hd)[0, :4, 0, :6].tolist()))
        _log({"debug": lines})
        print("\n".join(lines))
    return mx, float(d.nan_to_num(1e9).pow(2).mean().sqrt()), out


# (B, P, S, heads, head_dim, self_attn, varlen, weighted)
TC_CASES = [
    (4, 64, 132, 16, 80, True, False, False),      # BASELINE config 2, level 1: 196 keys, 2 S accumulators, 2 K/V stages
    (3, 16, 132, 16, 80, True, True, False),       # config 2, level 2: 16 queries in a 64-row tile
    (2, 256, 136, 16, 80, True, True, False),      # config 4, level 1: 392 keys
    (2, 64, 136, 16, 80, True, False, True),       # config 4, level 2 + attn_weights
    (5, 64, 20, 4, 80, False, True, False),        # cross-attention only, short ragged conditioning
    (2, 128, 7, 2, 80, True, False, False),        # two query tiles, odd conditioning length
    (160, 64, 132, 16, 80, True, False, False),    # more units than SMs: every CTA walks several units (ring wrap-around)
]


# <= 64 queries, <= 256 keys, no attn_weights: ragged key tiles, one key tile, the 256-key edge, many units
TT_CASES = [
    (6, 64, 100, 4, 80, True, True, False),        # ragged: some samples end inside key tile 0 (tile 1 fully masked), some in tile 1
    (3, 32, 12, 2, 80, True, False, False),        # one key tile (48 keys), 32 queries in the 64-wide N
    (2, 64, 190, 16, 80, True, True, False),       # 254 -> 256 keys: the largest tile set (single V stage)
    (300, 64, 132, 16, 80, True, True, False),     # ring wrap-around with ragged lengths (33 units per CTA)
]


@pytest.mark.parametrize("case", TC_CASES + TT_CASES)
def test_tcgen05_attention_vs_fp32_reference(case):
    """The default dispatch on every head_dim-80 shape of the workloads: the wgmma + TMA kernel."""
    mx, rms, _ = _run(*case)
    _log({"kernel": "wgmma", "case": case, "max_abs": mx, "rms": rms})
    assert mx < 4e-3 and rms < 4e-4, (case, mx, rms)      # outputs are O(1): fp16 P and fp16 output rounding


def test_tcgen05_row_major_kernel_on_the_transposed_kernels_shapes():
    """PB200_ATTN_MMA_SYNC=1 (child process) sends every head_dim-80 shape to the mma.sync kernel: the second kernel stays
    covered on the shapes the wgmma kernel normally takes."""
    here = os.path.dirname(os.path.abspath(__file__))
    cases = [c for c in TC_CASES + TT_CASES if not c[7]]
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_gpu_attention as t\n"
            "for c in %r:\n    mx, rms, _ = t._run(*c); print('RES', mx, rms)") % (os.path.dirname(here), here, cases)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, PB200_ATTN_MMA_SYNC="1"))
    assert r.returncode == 0, r.stderr[-2000:]
    res = [tuple(float(x) for x in l.split()[1:]) for l in r.stdout.splitlines() if l.startswith("RES")]
    assert len(res) == len(cases)
    for c, (mx, rms) in zip(cases, res):
        _log({"kernel": "mma.sync", "case": c, "max_abs": mx, "rms": rms})
        assert mx < 4e-3 and rms < 4e-4, (c, mx, rms)


@pytest.mark.parametrize("case", [(2, 64, 9, 4, 16, True, False, False), (2, 16, 20, 4, 32, True, True, True),
                                  (2, 100, 30, 2, 64, True, False, False), (3, 64, 132, 16, 80, True, True, False)])
def test_mma_sync_attention_vs_fp32_reference(case):
    """Other head dims run the mma.sync kernel; with PB200_ATTN_MMA_SYNC=1 (child process) so does head_dim 80."""
    if case[4] == 80:
        code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_gpu_attention as t; "
                "mx, rms, _ = t._run(*%r); print(mx, rms)") % (os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                               os.path.dirname(os.path.abspath(__file__)), case)
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, PB200_ATTN_MMA_SYNC="1"))
        assert r.returncode == 0, r.stderr[-2000:]
        mx, rms = (float(x) for x in r.stdout.split()[-2:])
    else:
        mx, rms, _ = _run(*case)
    _log({"kernel": "mma.sync", "case": case, "max_abs": mx, "rms": rms})
    assert mx < 4e-3 and rms < 4e-4, (case, mx, rms)
